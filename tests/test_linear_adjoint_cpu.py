"""The fused backward of a LinearField (csrc/tdq_linear_adjoint.cu) without a GPU: which adjoint problems take it, the
argument checks of its C entry points, and what ptxas makes of the kernel."""
import ctypes as C
import os
import re
import shutil
import subprocess
import types

import pytest
import torch

from torchdiffeq_b200 import LinearField, _lib
from torchdiffeq_b200.adjoint import fused_adjoint_weight
from torchdiffeq_b200.csrc import build

CPU = torch.device("cpu")


def _problem(func, shape=(64, 128), dtype=torch.float32, is_tuple=False):
    return types.SimpleNamespace(original_func=func, shape=None if is_tuple else torch.Size(shape), dtype=dtype,
                                 device=CPU, is_tuple=is_tuple)


class _Subclass(LinearField):
    def forward(self, t, y):
        return super().forward(t, y) * 2


def test_eligibility():
    W = torch.randn(128, 128)
    fp = LinearField(W.clone(), requires_grad=True)        # weight is a Parameter
    fb = LinearField(W.clone())                             # weight is a buffer
    on = {"fused_linear": True}
    assert fused_adjoint_weight(_problem(fp), (fp.weight,), on) is fp.weight
    assert fused_adjoint_weight(_problem(fb), (), on) is fb.weight
    assert fused_adjoint_weight(_problem(fp), (), on) is fp.weight          # W not differentiated: no W product
    assert fused_adjoint_weight(_problem(fp, shape=(7, 3, 128)), (fp.weight,), on) is fp.weight
    extra = torch.nn.Parameter(torch.zeros(3))
    refused = [
        (_problem(fp), (fp.weight,), {}),                                  # opt-in: the autograd backward is the default
        (_problem(fp), (fp.weight,), {"fused_linear": False}),
        (_problem(fp), (fp.weight, extra), on),                            # an extra adjoint parameter
        (_problem(fp), (extra,), on),
        (_problem(fp), (fp.weight,), dict(on, process_group=True)),        # the sharded backward stays generic
        (_problem(fp, is_tuple=True), (fp.weight,), on),                   # tuple state
        (_problem(fp, dtype=torch.float64), (fp.weight,), on),
        (_problem(LinearField(torch.randn(64, 64)), shape=(8, 64)), (), on),  # D != 128
        (_problem(_Subclass(W.clone())), (), on),                          # forward is not LinearField.forward
        (_problem(lambda t, y: y), (), on),
    ]
    for p, params, opts in refused:
        assert fused_adjoint_weight(p, params, opts) is None, (params, opts)
    f64 = LinearField(W.double())
    assert fused_adjoint_weight(_problem(f64, dtype=torch.float64), (), on) is None


def test_entry_points():
    lib = _lib.load()
    assert lib.tdq_linear_adjoint_supported(_lib.TDQ_F32, 128) == 1
    assert lib.tdq_linear_adjoint_supported(_lib.TDQ_F64, 128) == 0
    assert lib.tdq_linear_adjoint_supported(_lib.TDQ_F32, 64) == 0
    # one 128 x 128 float32 partial per chunk of 512 rows
    assert [lib.tdq_linear_adjoint_partials_len(r) for r in (0, 1, 512, 513, 65536)] == [0, 1 << 14, 1 << 14, 2 << 14,
                                                                                           128 << 14]


def test_entry_point_refusals():
    """Every refusal happens on the host, before anything is launched (no device is touched)."""
    lib = _lib.load()
    sc = (C.c_float * 3)(1.0, -1.0, -1.0)
    ok = 4096                               # a stand-in 16-byte aligned address, never dereferenced

    def refused(msg, **kw):
        args = dict(dtype=0, y=ok, a=ok, pw=ok, pwt=ok, width=128, rows=16, oy=ok, oa=ok, ow=ok, sc=sc, part=ok)
        args.update(kw)
        rc = lib.tdq_linear_adjoint_field(args["dtype"], args["y"], args["a"], args["pw"], args["pwt"], args["width"],
                                          args["rows"], args["oy"], args["oa"], args["ow"], args["sc"], args["part"], None)
        assert rc != 0
        assert msg in lib.tdq_last_error().decode()

    refused("null argument", y=None)
    refused("null argument", a=None)
    refused("null argument", pwt=None)
    refused("null argument", oa=None)
    refused("null argument", sc=None)
    refused("float32, width 128", dtype=1)
    refused("float32, width 128", width=64)
    refused("partials", part=None)
    refused("16-byte aligned", y=ok + 4)
    refused("16-byte aligned", ow=ok + 8)
    refused("16-byte aligned", part=ok + 4)
    refused("too many rows", rows=1 << 31)
    # no rows and no weight gradient: nothing to do, nothing launched
    assert lib.tdq_linear_adjoint_field(0, ok, ok, ok, ok, 128, 0, ok, ok, None, sc, None, None) == 0


NVCC = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CUOBJDUMP = shutil.which("cuobjdump") or os.path.join(os.path.dirname(NVCC), "cuobjdump")
KERNELS = {"with_w": "k_linear_adjointILb1E", "without_w": "k_linear_adjointILb0E"}
_INSN = re.compile(r"^\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P[T0-9]+\s+)?([A-Z][A-Z0-9_]*)(\S*)")


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    if not (os.path.exists(NVCC) and os.path.exists(CUOBJDUMP)):
        pytest.skip("nvcc / cuobjdump not available")
    obj = str(tmp_path_factory.mktemp("adjoint_sass") / "tdq_linear_adjoint.o")
    cmd = [NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(build.HERE, "tdq_linear_adjoint.cu"), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    sass = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


@pytest.mark.parametrize("which", sorted(KERNELS))
def test_adjoint_kernel_sass(compiled, which):
    """Both instantiations issue HGMMA (with W: the m64n128 products of a^T y too) and neither spills to local memory."""
    log, sass = compiled
    blocks = re.split(r"ptxas info\s+: Compiling entry function ", log)
    entry = [b for b in blocks[1:] if KERNELS[which] in b.split("\n", 1)[0]]
    assert len(entry) == 1
    m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", entry[0])
    assert m and (int(m.group(1)), int(m.group(2))) == (0, 0), entry[0]
    parts = re.split(r"\n\s*Function : ", sass)
    fn = [q for q in parts[1:] if KERNELS[which] in q.split("\n", 1)[0]]
    assert len(fn) == 1
    ops = [m.group(1) + m.group(2) for m in map(_INSN.match, fn[0].splitlines()) if m]
    assert any(op.startswith("HGMMA") for op in ops)
    assert not [op for op in ops if op.startswith(("LDL", "STL"))]
    wide = [line for line in fn[0].splitlines() if "HGMMA.64x128x16" in line]
    assert len(wide) == (6 if which == "with_w" else 0), len(wide)
