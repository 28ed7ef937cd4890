"""Whole sharded solves through the peer exchange on one GPU: rank `rank` of two whose peer holds an exact copy of its rows.

Every partial then arrives twice and 0 + s + s = 2s is exact; the element counts are doubled as well, so 2s / 2c is the
same rounded quotient as s / c.  Such a sharded solve is the unsharded solve of the shard, so it must equal that solve bit
for bit: solution, n_accept, n_reject and the last dt.

The peer is played by a proxy on the engine's library: its tdq_controller first enqueues, on the current stream, a copy of
norm_out into the own buffer's peer row and the peer's flag -- exactly what the peer's controller would store -- and then
forwards the call, so the kernel's wait ends on its first read.  The initial step's norms go through reduce_fn, which
doubles them.  Attempts are counted from arm(); halted trailing attempts tick the count too.  Only drivers that return to
the host for every attempt can be driven this way (lock step and eager); a captured graph would freeze the flag."""
import ctypes as C

import pytest
import torch

from test_gpu_exchange_kernels import NB, SENT, _flag, _image, _slot
from test_gpu_kernels import _same_bits
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import AdaptiveEngine, SolverFailure

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DRIVERS = {"lockstep": 0, "eager": 2}                            # run_ahead with graph=False


def _offsets():
    """Byte offsets of vals[p][r][0] and flags[p][r] in a buffer, from the ctypes mirror."""
    x = _lib.XBuf()
    base = C.addressof(x)
    vals = lambda p, r: C.addressof(x.vals[p][r]) - base
    flag = lambda p, r: C.addressof(x.flags[p]) - base + r * C.sizeof(C.c_uint64)
    return vals, flag


class _Proxy:
    """The engine's library with tdq_controller routed through the mirror."""

    def __init__(self, lib, mirror):
        self._lib, self._mirror = lib, mirror

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def tdq_controller(self, *args):
        return self._mirror.controller(*args)


class _Mirror:
    """The exchange object of AdaptiveEngine for rank `rank` of two, the peer holding a copy of this rank's rows."""

    def __init__(self, rank):
        self.rank, self.epoch, self.seq, self.sent = rank, 0, 0, []
        self.own = torch.full((NB,), SENT, dtype=torch.uint8, device=DEV)
        self.peer = torch.full((NB,), SENT, dtype=torch.uint8, device=DEV)
        self.eng = None

    def attach(self, eng):
        self.eng, self.lib = eng, eng.lib
        eng.lib = _Proxy(eng.lib, self)

    def arm(self, ctrl_ptr, stream):
        self.epoch += 1
        self.seq, self.sent = 0, []
        bufs = [self.own, self.peer] if self.rank == 0 else [self.peer, self.own]
        _lib.check(self.lib.tdq_ctrl_set_exchange(ctrl_ptr, _lib.ptr_array([b.data_ptr() for b in bufs]), self.rank, 2,
                                                  self.epoch, stream))

    def controller(self, ctrl, dc, norm_in, cnt, n_seg, ratio_dev, stream):
        norm = self.eng.norm_out
        assert norm_in == norm.data_ptr() and ratio_dev is None and n_seg + 1 == norm.numel()
        vals, flag = _offsets()
        par, other = _slot(self.epoch, self.seq), 1 - self.rank
        nv = min(n_seg + 1, _lib.TDQ_MAX_SEGS + 2)
        v0 = vals(par, other) // 8
        self.own.view(torch.float64)[v0:v0 + nv].copy_(norm[:nv])              # the peer's partials: a copy of ours
        f0 = flag(par, other) // 8
        self.own.view(torch.int64)[f0:f0 + 1].fill_(_flag(self.epoch, self.seq))
        self.sent.append(norm.clone())
        self.seq += 1
        return self.lib.tdq_controller(ctrl, dc, norm_in, cnt, n_seg, ratio_dev, stream)

    def check_last_partials(self, n_attempts):
        """The peer's buffer holds this rank's partials and flag of the last two attempts that exchanged (every attempt
        that did work does, and they come first), and its sentinel in every slot no attempt of this solve used."""
        x = _image(self.peer)
        for seq in range(max(0, n_attempts - 2), n_attempts):
            par = _slot(self.epoch, seq)
            assert x.flags[par][self.rank] == _flag(self.epoch, seq), seq
            got = torch.tensor(list(x.vals[par][self.rank][:self.sent[seq].numel()]), dtype=torch.float64)
            assert _same_bits(got, self.sent[seq]), seq
        assert all(x.flags[p][1 - self.rank] == int.from_bytes(bytes([SENT]) * 8, "little") for p in range(4))


def _problem(n, dtype, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = (0.2 + 2.8 * torch.rand(n, generator=g, dtype=torch.float64)).to(dtype).to(DEV)
    y0 = torch.randn(n, generator=g, dtype=torch.float64).to(dtype).to(DEV)

    def fn(t, y):
        return -a * y + torch.sin(3 * t + y)
    return fn, y0


def _pair(fn, n, dtype, method, rank, driver, segs=None, **kw):
    """(plain engine, sharded engine with its mirror) of the same problem."""
    counts = [int(l) for _, l in segs] if segs is not None else [n]
    common = dict(segs=segs, graph=False, device_loop=False, run_ahead=DRIVERS[driver], **kw)
    plain = AdaptiveEngine(fn, n, dtype, DEV, method, **common)
    mirror = _Mirror(rank)
    sharded = AdaptiveEngine(fn, n, dtype, DEV, method, reduce_fn=lambda b: b.mul_(2.0), n_global=2 * sum(counts),
                             seg_counts_global=[2 * c for c in counts], exchange=mirror, **common)
    mirror.attach(sharded)
    return plain, sharded, mirror


def _tols(dtype):
    return dict(rtol=1e-6, atol=1e-8) if dtype == torch.float64 else dict(rtol=1e-4, atol=1e-6)


def _solve_both(plain, sharded, mirror, y0, t64, driver):
    want = plain.solve(y0, t64).clone()
    got = sharded.solve(y0, t64).clone()
    assert sharded.driver == plain.driver == driver
    assert _same_bits(got, want)
    assert (sharded.n_accept, sharded.n_reject) == (plain.n_accept, plain.n_reject)
    assert sharded.mbox_host.contents.dt == plain.mbox_host.contents.dt
    assert mirror.seq >= sharded.n_attempts
    mirror.check_last_partials(sharded.n_attempts)
    return plain


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("method", ["dopri5", "dopri8", "tsit5", "bosh3"])
def test_mirrored_solve(method, dtype, rank, t_sign, driver):
    """Forward and reverse time, the initial step chosen by the solver (its norms through reduce_fn)."""
    n = 1000
    fn, y0 = _problem(n, dtype)
    plain, sharded, mirror = _pair(fn, n, dtype, method, rank, driver, t_sign=t_sign, **_tols(dtype))
    t64 = torch.linspace(0.0, 1.5, 4, dtype=torch.float64, device=DEV)
    _solve_both(plain, sharded, mirror, y0, t64, driver)
    assert plain.n_accept >= 4


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_mirrored_segments_vector_tolerances(dtype, rank, driver):
    """A state of three norm segments with gaps between them, per-element float64 tolerances."""
    n, segs = 1000, [(0, 300), (304, 400), (708, 292)]
    fn, y0 = _problem(n, dtype, seed=1)
    g = torch.Generator().manual_seed(5)
    rv = (1e-5 * (1 + torch.rand(n, generator=g, dtype=torch.float64))).to(DEV)
    av = (1e-7 * (1 + torch.rand(n, generator=g, dtype=torch.float64))).to(DEV)
    plain, sharded, mirror = _pair(fn, n, dtype, "dopri5", rank, driver, segs=segs, rtol=0.0, atol=0.0, rtol_vec=rv,
                                   atol_vec=av)
    t64 = torch.linspace(0.0, 1.0, 3, dtype=torch.float64, device=DEV)
    _solve_both(plain, sharded, mirror, y0, t64, driver)


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("method,whole", [("dopri5", True), ("tsit5", False)])
def test_mirrored_linear_field(method, whole, rank, driver):
    """A linear field on the tensor cores: dopri5 as the whole-attempt kernel with the norm folded in, tsit5 through the
    per-stage kernel and the separate norm."""
    width, rows = 128, 40
    n = width * rows
    g = torch.Generator().manual_seed(3)
    w = (-0.5 * torch.eye(width) + 0.05 * torch.randn(width, width, generator=g)).to(DEV)
    y0 = torch.randn(n, generator=g).to(DEV)
    fn = lambda t, y: (y.view(rows, width) @ w.T).reshape(-1)
    plain, sharded, mirror = _pair(fn, n, torch.float32, method, rank, driver, rtol=1e-5, atol=1e-7)
    for eng in (plain, sharded):
        assert eng.set_linear(w)
        assert eng.linear["whole"] == whole and eng.linear["fold"] == whole
    t64 = torch.linspace(0.0, 2.0, 3, dtype=torch.float64, device=DEV)
    _solve_both(plain, sharded, mirror, y0, t64, driver)


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_mirrored_rejects(dtype, rank, driver):
    """A first step far too large: the solve rejects before it accepts."""
    n = 1000
    fn, y0 = _problem(n, dtype, seed=2)
    plain, sharded, mirror = _pair(fn, n, dtype, "dopri5", rank, driver, first_step=0.9, **_tols(dtype))
    t64 = torch.linspace(0.0, 1.0, 3, dtype=torch.float64, device=DEV)
    _solve_both(plain, sharded, mirror, y0, t64, driver)
    assert sharded.n_reject > 0


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("rank", [0, 1])
def test_mirrored_three_solves(rank, driver):
    """Three solves on one engine: epochs 1, 2, 3 -- both parities, and the first parity used again."""
    n, dtype = 1000, torch.float64
    fn, y0 = _problem(n, dtype, seed=4)
    plain, sharded, mirror = _pair(fn, n, dtype, "tsit5", rank, driver, **_tols(dtype))
    for i in range(3):
        t64 = torch.linspace(0.0, 0.5 + 0.25 * i, 3 + i, dtype=torch.float64, device=DEV)
        _solve_both(plain, sharded, mirror, y0 * (1.0 + 0.5 * i), t64, driver)
        assert mirror.epoch == i + 1


@pytest.mark.parametrize("driver", list(DRIVERS))
@pytest.mark.parametrize("rank", [0, 1])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_mirrored_nonfinite(dtype, rank, driver):
    """A NaN enters y1 part-way: the sharded solve fails with the unsharded solve's exact error, after the same
    attempts."""
    n = 1000
    fn0, y0 = _problem(n, dtype, seed=6)
    nan = torch.tensor(float("nan"), dtype=dtype, device=DEV)
    fn = lambda t, y: torch.where(t > 0.3, nan, fn0(t, y))
    plain, sharded, mirror = _pair(fn, n, dtype, "dopri5", rank, driver, **_tols(dtype))
    t64 = torch.linspace(0.0, 1.0, 3, dtype=torch.float64, device=DEV)
    errs = []
    for eng in (plain, sharded):
        with pytest.raises(SolverFailure) as e:
            eng.solve(y0, t64)
        errs.append(str(e.value))
    assert errs[0] == errs[1]
    mp, ms = plain.mbox_host.contents, sharded.mbox_host.contents
    assert (ms.n_accept, ms.n_reject, ms.status) == (mp.n_accept, mp.n_reject, mp.status) and mp.n_accept > 0
    mirror.check_last_partials(int(ms.n_accept + ms.n_reject))


@pytest.mark.parametrize("rank", [0, 1])
def test_mirrored_too_many_segments(rank):
    """More norm segments than the exchange carries: the sharded solve fails with the error that names the limit and
    writes nothing to its peer, while the unsharded solve of the same state runs as usual."""
    n, segs = 650, [(10 * i, 10) for i in range(65)]
    fn, y0 = _problem(n, torch.float64, seed=7)
    plain, sharded, mirror = _pair(fn, n, torch.float64, "dopri5", rank, "lockstep", segs=segs, rtol=1e-6, atol=1e-8)
    t64 = torch.linspace(0.0, 0.5, 2, dtype=torch.float64, device=DEV)
    plain.solve(y0, t64)
    assert plain.n_accept > 0
    with pytest.raises(_lib.TdqError, match="at most 64 norm segments"):
        sharded.solve(y0, t64)
    assert mirror.seq == 1
    assert bytes(_image(mirror.peer)) == bytes([SENT]) * NB
