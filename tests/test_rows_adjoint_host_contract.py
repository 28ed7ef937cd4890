"""CPU checks of odeint_adjoint for independent rows: every refusal happens before any user code runs (and before the
device is touched), the new C entry points refuse null pointers and out-of-range shapes (every pointer is fake), and the
new kernels keep no stack frame and do not spill."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

import torchdiffeq_b200 as tdq

KEY = {"independent_rows": True}
SEMI = {"norm": "seminorm"}


@pytest.fixture(scope="module")
def lib():
    from torchdiffeq_b200.csrc import build
    build.build()
    from torchdiffeq_b200 import _lib
    return _lib


class Counting(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.calls = 0

    def forward(self, t, y):
        self.calls += 1
        return -y


def _refused(exc, match, options=KEY, adjoint_options=SEMI, f=None, y0=None, t=None, **kw):
    f = Counting() if f is None else f
    y0 = torch.ones(4, 3, requires_grad=True) if y0 is None else y0
    t = torch.tensor([0.0, 1.0]) if t is None else t
    with pytest.raises(exc, match=match):
        tdq.odeint_adjoint(f, y0, t, options=options, adjoint_options=adjoint_options, **kw)
    assert getattr(f, "calls", 0) == 0


def test_the_seminorm_is_required():
    for ao in (None, {}, {"norm": "default"}, {"norm": lambda x: x.abs().max()}):
        _refused(NotImplementedError, r"independent_rows.*adjoint_options=\{'norm': 'seminorm'", adjoint_options=ao)


def test_refusals_before_user_code():
    ni = NotImplementedError
    _refused(ni, "independent_rows.*differentiable", options=dict(KEY, differentiable=True))
    _refused(ValueError, "adjoint_options\\['independent_rows'\\] must be True",
             adjoint_options=dict(SEMI, independent_rows=False))
    _refused(ni, "independent_rows.*tuple states", y0=(torch.ones(4, 3), torch.ones(4, 3)))
    _refused(ni, "independent_rows.*event_fn", event_fn=lambda t, y: y.sum(-1))
    for name in ("step_t", "jump_t"):
        _refused(ni, "independent_rows.*%s" % name, options=dict(KEY, **{name: torch.tensor([0.5])}))
        _refused(ni, "independent_rows.*%s" % name, adjoint_options=dict(SEMI, **{name: torch.tensor([0.5])}))
    _refused(ni, "independent_rows.*process_group", options=dict(KEY, process_group=object()))
    _refused(ni, "independent_rows.*process_group", adjoint_options=dict(SEMI, process_group=object()))
    _refused(ni, "independent_rows.*compact_rows", options=dict(KEY, compact_rows=True))
    _refused(ni, "independent_rows.*compact_rows", adjoint_options=dict(SEMI, compact_rows=True))
    _refused(ni, "independent_rows.*fused_linear", adjoint_options=dict(SEMI, fused_linear=True))
    for m in ("rk4", "explicit_adams", "implicit_euler"):
        _refused(ni, "independent_rows.*adjoint_method", adjoint_method=m)
    _refused(ni, "independent_rows.*method", method="rk4")
    _refused(ni, "independent_rows.*tolerances", rtol=(1e-6,))
    _refused(ni, "independent_rows.*tolerances", adjoint_atol=torch.full((4, 3), 1e-8))
    for name in ("callback_step", "callback_accept_step_adjoint"):
        f = Counting()
        setattr(f, name, lambda t0, y0, dt: None)
        _refused(ni, "independent_rows.*callbacks", f=f)


def test_adjoint_method_still_needs_adjoint_options():
    """The reference's rule (adjoint.py:174-176) holds: with options given, a different adjoint_method needs
    adjoint_options -- which independent rows need anyway for the seminorm."""
    _refused(NotImplementedError, "independent_rows", adjoint_options=None, adjoint_method="bosh3")


def test_launchers_refuse_bad_arguments(lib):
    L = lib.load()
    fake = C.c_void_p(0x1000)
    sg = lib.RowsSegs()
    sg.n_seg, sg.offset[0], sg.len[0] = 1, 0, 4
    good = C.byref(sg)

    def bad(rc):
        assert rc != 0

    bad(L.tdq_rows_seg_sumsq(None, fake, 0, good, fake, None, 2, 4, fake, fake, None))
    bad(L.tdq_rows_seg_sumsq(fake, fake, 0, None, fake, None, 2, 4, fake, fake, None))
    bad(L.tdq_rows_seg_sumsq(fake, fake, 0, good, fake, None, 0, 4, fake, fake, None))
    bad(L.tdq_rows_seg_sumsq(fake, fake, 0, good, fake, None, 2, 3, fake, fake, None))      # segment past the row
    for n, off, ln in ((0, 0, 1), (5, 0, 1), (1, -1, 2), (1, 0, 0)):
        s = lib.RowsSegs()
        s.n_seg, s.offset[0], s.len[0] = n, off, ln
        bad(L.tdq_rows_seg_sumsq(fake, fake, 0, C.byref(s), fake, None, 2, 4, fake, fake, None))
        assert L.tdq_rows_seg_partials_len(2, C.byref(s)) == 0
    bad(L.tdq_rows_seg_error_norm_commit(fake, fake, 0, good, fake, None, fake, 2, 4, fake, fake, None))
    bad(L.tdq_rows_seg_initial_h0(fake, fake, 0, good, fake, None, 2, 4, None))
    bad(L.tdq_rows_seg_initial_finish(fake, fake, 0, good, None, 2, 4, None))
    bad(L.tdq_rows_seg_prepare(None, fake, 0, good, None, 2, 4, None))
    bad(L.tdq_rows_seg_controller(fake, fake, 0, good, None, 2, 4, None))
    bad(L.tdq_rows_seg_controller(fake, fake, 0, good, fake, 2, 3, None))
    # the augmented layout: o_y >= 1, adj_y after y, both inside the row
    bad(L.tdq_rows_adjoint_pack(0, None, None, None, fake, 2, 3, 4, 7, 10, None))
    bad(L.tdq_rows_adjoint_pack(0, fake, None, None, fake, 2, 3, 0, 7, 10, None))
    bad(L.tdq_rows_adjoint_pack(0, fake, None, None, fake, 2, 3, 4, 6, 10, None))
    bad(L.tdq_rows_adjoint_pack(0, fake, None, None, fake, 2, 3, 4, 7, 9, None))
    bad(L.tdq_rows_adjoint_handover(0, None, None, None, None, None, None, 2, 3, 4, 7, 10, None))
    bad(L.tdq_rows_adjoint_handover(0, fake, fake, None, None, None, None, 2, 3, 4, 7, 10, None))
    bad(L.tdq_rows_adjoint_handover(0, fake, None, None, fake, fake, None, 2, 3, 4, 7, 10, None))
    bad(L.tdq_rows_adjoint_handover(0, fake, None, None, None, None, None, 0, 3, 4, 7, 10, None))
    bad(L.tdq_rows_adjoint_weights(fake, fake, 0, fake, 0, fake, fake, fake, fake, 2, None))
    bad(L.tdq_rows_adjoint_weights(fake, fake, 0, fake, 18, fake, fake, fake, fake, 2, None))
    bad(L.tdq_rows_adjoint_weights(fake, fake, 0, None, 7, fake, fake, fake, fake, 2, None))
    bad(L.tdq_rows_adjoint_scale(fake, fake, 0, fake, fake, 7, None, fake, fake, 2, 3, 4, 7, 10, None))
    bad(L.tdq_rows_adjoint_scale(fake, fake, 0, fake, fake, 7, fake, fake, fake, 2, 3, 4, 7, 9, None))
    bad(L.tdq_rows_adjoint_scale(fake, fake, 0, fake, fake, 0, fake, fake, fake, 2, 3, 4, 7, 10, None))


NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
KERNELS = [k % t for t in ("f", "d") for k in (
    "k_rows_normI%sLi0ELb0ELb1E", "k_rows_normI%sLi1ELb0ELb1E", "k_rows_normI%sLi2ELb0ELb1E", "k_rows_h0I%sLb1E",
    "k_rows_finishI%sLb1E", "k_rows_prepareI%sLb1E", "k_rows_controllerI%sLb0ELb1E", "k_rows_adjoint_packI%sE",
    "k_rows_adjoint_handoverI%sE", "k_rows_adjoint_weightsI%sE", "k_rows_adjoint_scaleI%sE")]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip("nvcc not available")
    from torchdiffeq_b200.csrc import build
    obj = str(tmp_path_factory.mktemp("rows_adjoint") / "tdq_rows.o")
    r = subprocess.run([NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.HERE, "tdq_rows.cu"),
                        "-o", obj], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("kernel", KERNELS)
def test_kernels_do_not_spill(ptxas_log, kernel):
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", ptxas_log)
    hits = [b for b in blocks[1:] if kernel in b.split("\n", 1)[0]]
    assert len(hits) == 1, kernel
    assert re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", hits[0]), hits[0]
    assert re.search(r"Used (\d+) registers", hits[0]), hits[0]
