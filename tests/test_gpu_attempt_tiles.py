"""The whole-attempt kernel (csrc/tdq_attempt.cu) at row counts around its 32-row tile: one partial tile alone, one full tile,
a full tile plus one row, and three tiles per SM plus a partial one ("96P+17", P the device's SM count: CTA 0 runs four
tiles, the last of them partial, and every other CTA three).  Each k_i, y1, the error prefix and the
committed candidates must be BITWISE what the 16-row stage kernel (csrc/tdq_linear.cu) writes, and the squared error norm
agree to float64 summation order."""
import ctypes as C

import pytest
import torch

import grid_stride as G
from oracle import ode_oracle as O
from test_gpu_kernels import _engine, _rand
from test_gpu_linear import DEV, _attempt_reference, _planes, _weight

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("size", [31, 32, 33, "96P+17"])
def test_attempt_tile_boundaries_equal_stage_sequence(method, size):
    P = G.sm_count()
    rows = G.rows(size, P)
    if size == "96P+17":
        assert G.multi_tile(rows, P)
    n = rows * 128
    eng, _lib, _stream = _engine(method, torch.float32, n, 0.0371, 0.5, 1.0)
    lib = eng.lib
    S = O.tableau(method)["n_stages"]
    planes = _planes(lib, _lib, _weight(seed=5), _stream)
    y0 = _rand(n, torch.float32, 3).to(DEV)
    k0 = _rand(n, torch.float32, 4).to(DEV)
    ks, y1, er, norm, ycand, kcand = _attempt_reference(eng, _lib, _stream, planes, y0, k0, n, S)
    outs = [None] + [torch.full((n,), float("nan"), device=DEV) for _ in range(S)]
    y1a = torch.full((n,), float("nan"), device=DEV)
    era = torch.full((n,), float("nan"), device=DEV)
    for b in eng.ybuf + eng.kbuf:
        b.fill_(float("nan"))
    eng.norm_out.fill_(-1.0)
    kp = _lib.ptr_array([None] + [o.data_ptr() for o in outs[1:]])
    _lib.check(lib.tdq_linear_attempt(eng.ctrl.data_ptr(), C.byref(eng.tab), 0, kp, y1a.data_ptr(), era.data_ptr(),
                                      y0.data_ptr(), k0.data_ptr(), planes.data_ptr(), 128, n, eng.partials.data_ptr(),
                                      eng.norm_out.data_ptr(), None, 1, _stream()))
    torch.cuda.synchronize()
    for i in range(1, S + 1):
        assert torch.equal(outs[i], ks[i]), (method, rows, "k", i, float((outs[i] - ks[i]).abs().max()))
    assert torch.equal(y1a, y1) and torch.equal(era, er)
    assert torch.equal(eng.ybuf[1], ycand) and torch.equal(eng.kbuf[1], kcand)
    got = eng.norm_out.clone()
    assert abs(float(got[0]) - float(norm[0])) <= 1e-12 * abs(float(norm[0])), (float(got[0]), float(norm[0]))
    assert float(got[1]) == float(norm[1]) == 0.0
