"""The row-compaction kernels of tdq_rows.cu one launch at a time: tdq_rows_compact against torch.nonzero (padding, header
words, determinism, the resume of a paused solve), tdq_rows_gather / tdq_rows_scatter bitwise against torch indexing,
with row lengths that exercise scalar tails, several units per row and unaligned row starts."""
import pytest
import torch

from torchdiffeq_b200 import _lib

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda")
HDR_THRESHOLD, HDR_RUNNING, HDR_LISTED, HDR_PAUSED = 4, 5, 6, 7


def _st():
    return torch.cuda.current_stream().cuda_stream


def _rows(L, B):
    rows = torch.zeros(L.tdq_rows_size(B), dtype=torch.uint8, device=DEV)
    o = L.tdq_rows_offset(_lib.ROWS_DONE, B)
    return rows, rows[o:o + 4 * B].view(torch.int32), rows[:32].view(torch.int32)


def _ctrl(L):
    return torch.zeros(L.tdq_ctrl_size(), dtype=torch.uint8, device=DEV)


def _patterns(B):
    g = torch.Generator().manual_seed(B)
    yield "random", (torch.rand(B, generator=g) < 0.6).to(torch.int32)
    yield "all_done", torch.ones(B, dtype=torch.int32)
    yield "none_done", torch.zeros(B, dtype=torch.int32)
    one = torch.ones(B, dtype=torch.int32)
    one[B // 2] = 0
    yield "single_running", one
    if B > 1:
        last = torch.ones(B, dtype=torch.int32)
        last[-1] = 0
        yield "last_running", last


@pytest.mark.parametrize("B", [1, 31, 33, 1025, 65536])
def test_compact_matches_nonzero(B):
    L = _lib.load()
    rows, done, hdr = _rows(L, B)
    ctrl = _ctrl(L)
    for name, flags in _patterns(B):
        done.copy_(flags)
        running = torch.nonzero(flags == 0).view(-1)
        n = running.numel()
        for size in sorted({B, max(n, 1), (B + 1) // 2 if n <= (B + 1) // 2 else B}):
            thr = size // 2 if size > 1 else 0
            outs = []
            for _ in range(2):
                idx = torch.full((size,), -7, dtype=torch.int64, device=DEV)
                _lib.check(L.tdq_rows_compact(ctrl.data_ptr(), rows.data_ptr(), idx.data_ptr(), B, size, thr, _st()))
                outs.append(idx.cpu())
            assert torch.equal(outs[0], outs[1]), name                          # the same flags, the same list
            idx, h = outs[0], hdr.cpu()
            assert torch.equal(idx[:n], running), (name, size)
            assert torch.equal(idx[n:], torch.full((size - n,), int(running[-1]) if n else 0, dtype=torch.int64)), name
            assert int(h[HDR_LISTED]) == n and int(h[HDR_RUNNING]) == n and int(h[HDR_THRESHOLD]) == thr


def test_compact_resumes_only_a_paused_solve():
    """Without the pause flag the control block is not touched (a halted solve that is done or failed stays so); with it
    exactly one control word changes: halt, cleared."""
    L = _lib.load()
    B = 40
    rows, done, hdr = _rows(L, B)
    ctrl = _ctrl(L)
    ctrl.fill_(0xFF)
    idx = torch.zeros(B, dtype=torch.int64, device=DEV)
    done[:30] = 1
    _lib.check(L.tdq_rows_compact(ctrl.data_ptr(), rows.data_ptr(), idx.data_ptr(), B, 20, 10, _st()))
    assert bool((ctrl == 0xFF).all())
    hdr[HDR_PAUSED] = 1
    _lib.check(L.tdq_rows_compact(ctrl.data_ptr(), rows.data_ptr(), idx.data_ptr(), B, 20, 5, _st()))
    words = ctrl.view(torch.int32).cpu()
    assert int((words == 0).sum()) == 1 and int((words == -1).sum()) == words.numel() - 1
    h = hdr.cpu()
    assert int(h[HDR_PAUSED]) == 0 and int(h[HDR_THRESHOLD]) == 5 and int(h[HDR_LISTED]) == 10
    _lib.check(L.tdq_rows_set_compact_threshold(rows.data_ptr(), B, 3, _st()))
    assert int(hdr.cpu()[HDR_THRESHOLD]) == 3


def _index(B, size, seed):
    g = torch.Generator().manual_seed(seed)
    n = max(1, size - 3)
    run = torch.sort(torch.randperm(B, generator=g)[:n]).values
    return torch.cat([run, run[-1].repeat(size - n)]), n


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("D", [1, 3, 4, 1024, 1025, 4099])
def test_gather_scatter_bitwise(dtype, D):
    L = _lib.load()
    dc = _lib.TDQ_F32 if dtype == torch.float32 else _lib.TDQ_F64
    B = 37
    rows, done, hdr = _rows(L, B)
    ctrl = _ctrl(L)
    for size in (B, 19, 5, 1):
        idx_h, n = _index(B, size, D + size)
        g = torch.Generator().manual_seed(size)
        src = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        t_src = torch.randn(B, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        idx = idx_h.to(DEV)
        dst = torch.full((size, D), float("nan"), dtype=dtype, device=DEV)
        t_dst = torch.full((size,), float("nan"), dtype=dtype, device=DEV)
        _lib.check(L.tdq_rows_gather(dc, idx.data_ptr(), size, src.data_ptr(), t_src.data_ptr(), dst.data_ptr(),
                                     t_dst.data_ptr(), B, D, _st()))
        assert torch.equal(dst, src[idx]) and torch.equal(t_dst, t_src[idx])
        # scatter: only the listed rows, set by tdq_rows_compact from the DONE flags
        flags = torch.ones(B, dtype=torch.int32)
        flags[idx_h[:n]] = 0
        done.copy_(flags)
        lst = torch.zeros(size, dtype=torch.int64, device=DEV)
        _lib.check(L.tdq_rows_compact(ctrl.data_ptr(), rows.data_ptr(), lst.data_ptr(), B, size, 0, _st()))
        assert torch.equal(lst.cpu(), idx_h)
        res = torch.randn(size, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        full = torch.randn(B, D, generator=g, dtype=torch.float64).to(dtype).to(DEV)
        want = full.clone()
        want[idx_h[:n]] = res[:n]
        _lib.check(L.tdq_rows_scatter(rows.data_ptr(), dc, lst.data_ptr(), size, res.data_ptr(), full.data_ptr(), B, D,
                                      _st()))
        assert torch.equal(full, want)                                   # padding and unlisted rows untouched


def test_unaligned_bases_and_event_values():
    """Views whose first element is not 16-byte aligned take the scalar path; K-wide float64 event values scatter."""
    L = _lib.load()
    B, D = 29, 37
    rows, done, _ = _rows(L, B)
    ctrl = _ctrl(L)
    idx_h, n = _index(B, 11, 3)
    flags = torch.ones(B, dtype=torch.int32)
    flags[idx_h[:n]] = 0
    done.copy_(flags)
    idx = torch.zeros(11, dtype=torch.int64, device=DEV)
    _lib.check(L.tdq_rows_compact(ctrl.data_ptr(), rows.data_ptr(), idx.data_ptr(), B, 11, 0, _st()))
    base = torch.randn(B * D + 1, dtype=torch.float32, device=DEV)
    src = base[1:].view(B, D)
    out = torch.zeros(11 * D + 1, dtype=torch.float32, device=DEV)
    dst = out[1:].view(11, D)
    _lib.check(L.tdq_rows_gather(_lib.TDQ_F32, idx.data_ptr(), 11, src.data_ptr(), None, dst.data_ptr(), None, B, D,
                                 _st()))
    assert torch.equal(dst, src[idx])
    for K in (1, 3):
        val = torch.randn(11, K, dtype=torch.float64, device=DEV)
        ev = torch.randn(B, K, dtype=torch.float64, device=DEV)
        want = ev.clone()
        want[idx_h[:n]] = val[:n]
        _lib.check(L.tdq_rows_scatter(rows.data_ptr(), _lib.TDQ_F64, idx.data_ptr(), 11, val.data_ptr(), ev.data_ptr(), B,
                                      K, _st()))
        assert torch.equal(ev, want)
