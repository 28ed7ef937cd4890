"""CPU checks of the C ABI: the library builds/loads, exports every symbol include/tdq.h declares,
and its tableaus are the reference's float64 values (tests/golden/tableaus.json)."""
import json
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


def test_header_symbols_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "tdq.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = set(re.findall(r"\b(tdq_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    L = lib.load()
    missing = [n for n in declared if not hasattr(L, n)]
    assert not missing, missing
    # and the Python binding covers the whole header
    assert declared == set(lib.EXPORTED_SYMBOLS), declared ^ set(lib.EXPORTED_SYMBOLS)
    assert L.tdq_abi_version() == lib.ABI_VERSION == 2


def test_struct_sizes(lib):
    import ctypes as C
    L = lib.load()
    assert C.sizeof(lib.Tableau) == L.tdq_sizeof(0) == 16 + 8 * (16 + 16 * 17 + 3 * 17)
    assert C.sizeof(lib.Options) == L.tdq_sizeof(1)
    assert C.sizeof(lib.Mailbox) == L.tdq_sizeof(2)
    assert lib.load().tdq_ctrl_size() % 256 == 0
    assert lib.load().tdq_ctrl_tstage_offset() % 16 == 0


@pytest.mark.parametrize("name", ["dopri5", "dopri8", "tsit5", "bosh3", "fehlberg2", "adaptive_heun"])
def test_tableaus_match_reference(lib, name):
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "tableaus.json")))[name]
    got = lib.tableau_as_dict(name)
    for key in ("alpha", "beta", "c_sol", "c_err", "c_mid", "order", "fsal", "n_stages"):
        assert got[key] == ref[key], key      # bitwise: same float64 values


def test_unknown_tableau_is_an_error(lib):
    with pytest.raises(lib.TdqError):
        lib.tableau("rk45")


def test_no_cpu_fallback():
    import torch
    import torchdiffeq_b200 as tdq
    y0 = torch.ones(3)
    with pytest.raises(tdq.TdqError):
        tdq.odeint(lambda t, y: -y, y0, torch.tensor([0., 1.]))


def test_linear_attempt_host_side_contract():
    """tdq_linear_attempt_supported is a pure host function of (tableau, dtype, width); tdq_linear_attempt validates its
    arguments before it touches the device (csrc/tdq_attempt.cu)."""
    import ctypes as C
    from torchdiffeq_b200 import _lib
    lib = _lib.load()
    want = {"dopri5": 1, "bosh3": 1, "tsit5": 0, "dopri8": 0, "fehlberg2": 0, "adaptive_heun": 0}
    for m, w in want.items():
        tab = _lib.tableau(m)
        assert lib.tdq_linear_attempt_supported(C.byref(tab), 0, 128) == w, m
        assert lib.tdq_linear_attempt_supported(C.byref(tab), 1, 128) == 0          # float64
        assert lib.tdq_linear_attempt_supported(C.byref(tab), 0, 64) == 0           # another width
    assert lib.tdq_linear_attempt_supported(None, 0, 128) == 0
    tab = _lib.tableau("dopri5")
    bad = C.c_void_p(16)                                                             # never dereferenced: the checks come first
    kp = _lib.ptr_array([None] + [16] * 6)
    # null control block / float64 / state not a whole number of rows / norm outputs that do not go together /
    # the reserved seg_counts_dev not NULL, without and with the folded norm
    assert lib.tdq_linear_attempt(None, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, None, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 1, kp, bad, bad, None, None, bad, 128, 1280, None, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1281, None, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, bad, None, None, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, None, None, bad, 1, None) != 0
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 1280, bad, bad, bad, 1, None) != 0
    # a tableau the kernel does not take is refused as well
    t8 = _lib.tableau("dopri8")
    k8 = _lib.ptr_array([None] + [16] * 13)
    assert lib.tdq_linear_attempt(bad, C.byref(t8), 0, k8, bad, bad, None, None, bad, 128, 1280, None, None, None, 1, None) != 0
    # an empty state is a no-op that succeeds without a launch
    assert lib.tdq_linear_attempt(bad, C.byref(tab), 0, kp, bad, bad, None, None, bad, 128, 0, None, None, None, 1, None) == 0
