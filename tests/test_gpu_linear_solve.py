"""The persistent fused solve (tdq_linear_solve, k_linear_solve in csrc/tdq_attempt.cu) on the GPU.

A LinearField solve that the device-side loop would run (device_loop True / 'auto', run-ahead, the plain norm) runs all its
attempts, controller steps and interpolant fits in one launch.  It must give what the per-attempt path gives, bit for bit:
the solution, n_accept, n_reject and nfe, and the same failures with the same text.  The per-attempt path is what
device_loop=False runs (the host replays the captured attempt) and what lock step runs (run_ahead=0: exactly one attempt per
mailbox tick, so its nfe counts no trailing no-op attempts, like the device loop)."""
import pytest
import torch

import grid_stride as G
import problems as P

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RTOL, ATOL = 1e-5, 1e-7


def tdq():
    import torchdiffeq_b200
    return torchdiffeq_b200


def _weight():
    return P.skew_matrix(128, torch.float32).to(DEV)


def _y0(rows, seed=1):
    return torch.randn(rows, 128, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _solve(W, y0, t, method="dopri5", cache=False, **opts):
    st = {}
    opts.setdefault("device_loop", True)
    with torch.no_grad():
        out = tdq().odeint(tdq().LinearField(W), y0, t, method=method, rtol=RTOL, atol=ATOL,
                           options=dict(cache=cache, **opts), _stats=st)
    return out.clone(), st


def _persistent(st):
    """a fused solve that ran as one launch: the start-up's ten launches at most, + 1, whatever the number of attempts"""
    return bool(st["fused_attempt"]) and st["launches"] <= 11 and st["driver"] == "persistent"


def _same(a, b):
    out_a, st_a = a
    out_b, st_b = b
    assert torch.equal(out_a, out_b), float((out_a - out_b).abs().max())
    assert (st_a["n_accept"], st_a["n_reject"]) == (st_b["n_accept"], st_b["n_reject"])


def _check(W, y0, t, method="dopri5", **opts):
    got = _solve(W, y0, t, method, **opts)
    assert _persistent(got[1]), got[1]
    _same(got, _solve(W, y0, t, method, device_loop=False, **opts))
    lock = _solve(W, y0, t, method, run_ahead=0, **opts)
    _same(got, lock)
    assert got[1]["nfe"] == lock[1]["nfe"]
    return got


def _rows(size):
    """size (an int or tests/grid_stride.py's "aP+b") as a row count for this device.  "32P" gives every CTA exactly one
    full tile; every larger size gives at least one CTA two or more, so each CTA's partial covers several tiles."""
    P = G.sm_count()
    B = G.rows(size, P)
    if size == "32P":
        assert G.tiles(B) == P
    elif B > 32 * P:
        assert G.multi_tile(B, P)
    return B


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("rows", [1, 31, 32, 33, 1000, "32P", "32P+1", "64P+17", 65536])
def test_persistent_solve_bitwise(method, rows):
    _check(_weight(), _y0(_rows(rows)), torch.tensor([0.0, 2.0], device=DEV), method)


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_persistent_solve_reverse_time(method):
    _check(_weight(), _y0(33), torch.tensor([2.0, 0.5], device=DEV), method)


MANY_OUTPUTS = torch.cat([torch.linspace(0.0, 0.01, 7), torch.linspace(0.02, 3.0, 60)])


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
def test_persistent_solve_many_outputs(method):
    """outputs inside most steps, several inside one step: the in-kernel fit runs many times"""
    t = MANY_OUTPUTS.to(DEV)
    out, st = _check(_weight(), _y0(1000), t, method)
    assert out.shape[0] == t.numel()


@pytest.mark.parametrize("method", ["dopri5", "bosh3"])
@pytest.mark.parametrize("case", ["reverse_64P+17", "many_outputs_65536"])
def test_persistent_solve_several_tiles_per_cta(method, case):
    """reverse time with a partial tile in CTA 0's third pass, and the in-kernel fit (grid-stride over 8.4 M elements) at
    nearly every step of the benchmark's batch"""
    if case.startswith("reverse"):
        _check(_weight(), _y0(_rows("64P+17")), torch.tensor([2.0, 0.5], device=DEV), method)
    else:
        t = MANY_OUTPUTS.to(DEV)
        out, _ = _check(_weight(), _y0(_rows(65536)), t, method)
        assert out.shape[0] == t.numel()


def test_persistent_solve_reverse_many_outputs():
    _check(_weight(), _y0(65), torch.linspace(1.5, -0.5, 23).to(DEV), "dopri5")


def test_persistent_solve_first_step():
    _check(_weight(), _y0(64), torch.tensor([0.0, 1.0], device=DEV), "dopri5", first_step=0.01)


def test_persistent_solve_weight_changed_in_place():
    W = _weight()
    y0, t = _y0(96), torch.linspace(0.0, 1.0, 4).to(DEV)
    first = _solve(W, y0, t, cache=True)
    assert _persistent(first[1])
    W.mul_(0.5)
    second = _solve(W, y0, t, cache=True)
    assert _persistent(second[1])
    _same(second, _solve(W.clone(), y0, t, device_loop=False))
    assert not torch.equal(first[0], second[0])


def test_launches_do_not_grow_with_attempts():
    W, y0 = _weight(), _y0(256)
    short = _solve(W, y0, torch.tensor([0.0, 0.5], device=DEV))[1]
    long = _solve(W, y0, torch.tensor([0.0, 5.0], device=DEV))[1]
    assert long["attempts"] > short["attempts"] + 5
    assert long["launches"] == short["launches"]


@pytest.mark.parametrize("opts", [dict(device_loop=False), dict(run_ahead=0), dict(vector_atol=True)])
def test_other_modes_take_the_per_attempt_path(opts):
    opts = dict(opts)
    W, y0, t = _weight(), _y0(64), torch.tensor([0.0, 1.0], device=DEV)
    if opts.pop("vector_atol", False):
        st = {}
        with torch.no_grad():
            tdq().odeint(tdq().LinearField(W), y0, t, method="dopri5", rtol=RTOL, atol=torch.full_like(y0, ATOL),
                         options=dict(cache=False), _stats=st)
    else:
        st = _solve(W, y0, t, **opts)[1]
    assert st["launches"] > st["attempts"], st
    assert st["driver"] == ("lockstep" if opts.get("run_ahead") == 0 else "capture"), st


def _failure(W, y0, t, **opts):
    with pytest.raises(Exception) as e:
        _solve(W, y0, t, **opts)
    return type(e.value), str(e.value)


@pytest.mark.parametrize("case", ["max_num_steps", "dt_underflow", "nonfinite", "nonfinite_32P+5", "nonfinite_last"])
def test_persistent_solve_failures(case):
    """40 rows; and 65,536 with the infinity in row 32P + 5 (CTA 0's second tile) or in the last row"""
    W = _weight()
    y0 = _y0(_rows(65536) if case in ("nonfinite_32P+5", "nonfinite_last") else 40)
    t = torch.tensor([0.0, 2.0], device=DEV)
    opts = {}
    if case == "max_num_steps":
        opts["max_num_steps"] = 3
    elif case == "dt_underflow":
        t = torch.tensor([1.0, 2.0], device=DEV)
        opts["first_step"] = 1e-20                     # 1 + 1e-20 == 1: the first attempt fails
    else:
        r = {"nonfinite": 3, "nonfinite_32P+5": G.rows("32P+5", G.sm_count()), "nonfinite_last": y0.shape[0] - 1}[case]
        y0[r, 5] = float("inf")
        opts["first_step"] = 0.01                      # past the initial step selection, which would end in dt 0
    got = _failure(W, y0, t, **opts)
    assert got == _failure(W, y0, t, device_loop=False, **opts)
    assert got == _failure(W, y0, t, run_ahead=0, **opts)
    assert {"max_num_steps": "max_num_steps exceeded",
            "dt_underflow": "underflow in dt"}.get(case, "non-finite values") in got[1], got
