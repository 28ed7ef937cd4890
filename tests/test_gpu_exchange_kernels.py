"""The peer exchange of a sharded solve inside tdq_controller (csrc/tdq_ctrl.cu), one launch at a time on one GPU.

Rank `me` of R ranks is emulated in one process: R device buffers laid out as tdq_sizeof(3) / _lib.XBuf, every byte a
sentinel.  Before each launch the test writes what the other ranks' controllers would have stored into me's buffer --
their partials and their flag (epoch << 32) | (seq + 1) in slot ((epoch & 1) << 1) | (seq & 1) -- and checks that every
awaited flag is there, so the kernel's spin loop ends on its first read: nothing runs concurrently and nothing waits for
the 10 s timeout.  The mailbox must then equal, byte for byte, that of an unarmed (world-1) block fed the rank-order
float64 sum of the R vectors, and every peer buffer must hold this rank's partials and flag in that slot and its
sentinel everywhere else.

The partials make the order of the sum matter: per segment, rank 0 holds 2**53 u, ranks 1 .. R-2 hold u and rank R-1
holds w - 2**53 u (u a power of two, w a multiple of u).  In rank order each u is lost to round-to-even against 2**53 u
and the total is w; summed in any order that brings the u's together first it is w + (R - 2) u.  With R = 2 the order
cannot matter; R = 3 and R = 16 catch a wrong one.

Run as a script, this file is the second process of test_ipc_two_processes (rank 1 over CUDA IPC)."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_kernels import _engine
from torchdiffeq_b200 import _lib
from torchdiffeq_b200._engine import _stream

pytestmark = pytest.mark.gpu

SENT = 0xA5                                   # every byte of a fresh buffer; as a flag it is never awaited
U = 2.0 ** -6
BIG = 2.0 ** 53 * U
NB = C.sizeof(_lib.XBuf)


def _slot(epoch, seq):
    return ((epoch & 1) << 1) | (seq & 1)


def _flag(epoch, seq):
    return ((epoch << 32) | (seq + 1)) & (2 ** 64 - 1)


def _buffers(R):
    return [torch.full((NB,), SENT, dtype=torch.uint8, device="cuda") for _ in range(R)]


def _image(buf):
    """The buffer's bytes as an XBuf (after the stream's work)."""
    torch.cuda.synchronize()
    return _lib.XBuf.from_buffer_copy(buf.cpu().numpy().tobytes())


def _upload(buf, x):
    buf.copy_(torch.frombuffer(bytearray(bytes(x)), dtype=torch.uint8))
    torch.cuda.synchronize()


def _store(x, epoch, seq, r, vals):
    """What rank r's controller stores into a buffer for attempt `seq`: its partials, then its flag."""
    par = _slot(epoch, seq)
    for i, v in enumerate(vals[:_lib.TDQ_MAX_SEGS + 2]):
        x.vals[par][r][i] = v
    x.flags[par][r] = _flag(epoch, seq)


def _deliver(bufs, me, epoch, seq, parts):
    """Every other rank's store of attempt `seq` into me's buffer."""
    x = _image(bufs[me])
    for r, v in enumerate(parts):
        if r != me:
            _store(x, epoch, seq, r, v)
    _upload(bufs[me], x)


def _arm(eng, bufs, me, epoch):
    ptrs = _lib.ptr_array([b.data_ptr() for b in bufs])
    _lib.check(eng.lib.tdq_ctrl_set_exchange(eng.ctrl.data_ptr(), ptrs, me, len(bufs), epoch, _stream()))


def _launch(eng, bufs, me, epoch, norm_in, cnt, n_seg, ratio_dev=None):
    """One tdq_controller of rank `me` of len(bufs) ranks, after checking that every flag it may wait for is in its own
    buffer.  Returns the images of all buffers just before the launch; the mailbox has ticked when it returns."""
    mb = eng.mbox_host.contents
    seq = int(mb.seq)
    par, want = _slot(epoch, seq), _flag(epoch, seq)
    before = [_image(b) for b in bufs]
    missing = [t for t in range(len(bufs)) if t != me and before[me].flags[par][t] != want]
    assert not missing, ("flags not delivered before the launch", missing, seq)
    _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, norm_in.data_ptr(), cnt.data_ptr(), n_seg,
                                      ratio_dev.data_ptr() if ratio_dev is not None else None, _stream()))
    torch.cuda.synchronize()
    assert mb.seq == seq + 1
    return before


def _reference(eng, norm_in, cnt, n_seg, ratio_dev=None):
    """The same controller step on an unarmed block."""
    _lib.check(eng.lib.tdq_controller(eng.ctrl.data_ptr(), eng.dt_code, norm_in.data_ptr(), cnt.data_ptr(), n_seg,
                                      ratio_dev.data_ptr() if ratio_dev is not None else None, _stream()))
    torch.cuda.synchronize()
    return bytes(eng.mbox_host.contents)


def _partials(R, ks, bad=(0.0,)):
    """R vectors of len(ks) + 1 partials: segment s sums to ks[s] * U in rank order only (module docstring); slot n_seg
    (the non-finite count) is bad[r] for rank r (0 when not given)."""
    parts = []
    for r in range(R):
        if r == 0 and R > 1:
            v = [BIG] * len(ks)
        elif r == R - 1:
            v = [k * U - BIG for k in ks] if R > 1 else [k * U for k in ks]
        else:
            v = [U] * len(ks)
        parts.append(v + [bad[r] if r < len(bad) else 0.0])
    return parts


def _rank_order_sum(parts):
    out = []
    for i in range(len(parts[0])):
        a = 0.0
        for v in parts:
            a += v[i]
        out.append(a)
    return out


def _dev(v, dtype=torch.float64):
    return torch.tensor(v, dtype=dtype, device="cuda")


def _case(n_seg, outcome):
    """(counts, ks): ratio about 0.5 in every segment, and for a reject one segment at about 2."""
    counts = [3 + (7 * s) % 50 for s in range(n_seg)]
    ks = [16 * c + s % 8 for s, c in enumerate(counts)]
    if outcome == "reject":
        ks[n_seg // 2] = 256 * counts[n_seg // 2] + 1
    return counts, ks


def _expect_send(before, me, epoch, seq, vals):
    """The buffers after rank me's controller of attempt `seq` exchanged: its store in every one of them, nothing else."""
    after = [_lib.XBuf.from_buffer_copy(bytes(x)) for x in before]
    for x in after:
        _store(x, epoch, seq, me, vals)
    return after


def _assert_images(bufs, want, what):
    for t, (b, w) in enumerate(zip(bufs, want)):
        got = _image(b)
        assert bytes(got) == bytes(w), (what, t, _first_diff(got, w))


def _first_diff(got, want):
    for name in ("flags", "vals"):
        for p in range(4):
            for r in range(_lib.TDQ_MAX_RANKS):
                g, w = bytes(getattr(got, name)[p][r]), bytes(getattr(want, name)[p][r])
                if g != w:
                    return (name, p, r, list(getattr(got, name)[p][r])[:8], list(getattr(want, name)[p][r])[:8])
    return None


@pytest.mark.parametrize("t_sign", [1.0, -1.0])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("outcome", ["accept", "reject"])
@pytest.mark.parametrize("n_seg", [1, 4, 64])
@pytest.mark.parametrize("R", [2, 3, 16])
def test_receive_and_send(R, n_seg, outcome, dtype, t_sign):
    """Every rank `me` of R: the mailbox equals the world-1 block's fed the rank-order sum (so every rank decides the
    same), and each of the R buffers holds me's partials and flag in the attempt's slot and its sentinel elsewhere."""
    counts, ks = _case(n_seg, outcome)
    parts = _partials(R, ks)
    cnt = _dev(counts, torch.int64)
    dt, t0, epoch = 0.02, 0.5, 3
    ref = _engine("dopri5", dtype, 16, dt, t0, t_sign)[0]
    want_mb = _reference(ref, _dev(_rank_order_sum(parts)), cnt, n_seg)
    assert ref.mbox_host.contents.accept == (outcome == "accept")
    for me in range(R):
        eng = _engine("dopri5", dtype, 16, dt, t0, t_sign)[0]
        bufs = _buffers(R)
        _arm(eng, bufs, me, epoch)
        _deliver(bufs, me, epoch, 0, parts)
        before = _launch(eng, bufs, me, epoch, _dev(parts[me]), cnt, n_seg)
        assert bytes(eng.mbox_host.contents) == want_mb, me
        _assert_images(bufs, _expect_send(before, me, epoch, 0, parts[me]), ("send", me))


def _reinit(eng, dt, t0=0.5):
    """A new solve on the same control block and mailbox (what AdaptiveEngine._begin resets)."""
    mb = eng.mbox_host.contents
    mb.seq, mb.status, mb.done, mb.par, mb.accept, mb.n_accept, mb.n_reject = 0, 0, 0, 0, 0, 0, 0
    _lib.check(eng.lib.tdq_ctrl_init(eng.ctrl.data_ptr(), C.byref(eng.tab), C.byref(eng.opt), eng.t_out.data_ptr(), t0, 2,
                                     eng.mbox_dev, _stream()))
    _lib.check(eng.lib.tdq_set_first_step(eng.ctrl.data_ptr(), float(dt), _stream()))
    _lib.check(eng.lib.tdq_prepare_attempt(eng.ctrl.data_ptr(), eng.dt_code, None, _stream()))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("me", [0, 1, 2])
def test_slots_across_attempts_and_solves(me, dtype):
    """Three solves on one control block, armed with epochs e, e + 1, e + 2 (both parities, and a high bit that must
    survive into the flag), each several attempts of accepts and rejects, so that the attempt parity and the accepted
    pair's parity part ways.  After every attempt the mailbox equals the world-1 block's and the R buffers equal what
    the slot rule predicts -- with everything earlier attempts and solves left in the other slots."""
    R, n_seg, dt = 3, 4, 0.02
    e = (1 << 30) | 5
    eng = _engine("dopri5", dtype, 16, dt)[0]
    ref = _engine("dopri5", dtype, 16, dt)[0]
    bufs = _buffers(R)
    want = [_image(b) for b in bufs]
    pattern = {e: "ARRAAR", e + 1: "RAAR", e + 2: "ARA"}
    for epoch, steps in pattern.items():
        if epoch != e:
            _reinit(eng, dt)
            _reinit(ref, dt)
        _arm(eng, bufs, me, epoch)
        pars = set()
        for seq, step in enumerate(steps):
            counts, ks = _case(n_seg, "accept" if step == "A" else "reject")
            ks = [k + 3 * seq for k in ks]                             # a different sum every attempt
            parts = _partials(R, ks)
            cnt = _dev(counts, torch.int64)
            assert eng.mbox_host.contents.seq == seq
            _deliver(bufs, me, epoch, seq, parts)
            for r in range(R):
                if r != me:
                    _store(want[me], epoch, seq, r, parts[r])
            before = _launch(eng, bufs, me, epoch, _dev(parts[me]), cnt, n_seg)
            assert [bytes(x) for x in before] == [bytes(x) for x in want], (epoch, seq)
            want = _expect_send(want, me, epoch, seq, parts[me])
            mb_ref = _reference(ref, _dev(_rank_order_sum(parts)), cnt, n_seg)
            mb = eng.mbox_host.contents
            assert bytes(mb) == mb_ref, (epoch, seq)
            assert mb.accept == (step == "A"), (epoch, seq)
            pars.add((seq & 1, mb.par))
            _assert_images(bufs, want, (epoch, seq))
        if epoch == e:
            assert len(pars) >= 3                                      # attempt parity and pair parity do differ
    # the flags the last solve left, read through the mirror: (e + 2) << 32 | attempt + 1, in slots 2 (even) / 3 (odd)
    got = _image(bufs[(me + 1) % R])
    assert got.flags[2][me] == ((e + 2) << 32) | 3 and got.flags[3][me] == ((e + 2) << 32) | 2
    assert got.flags[0][me] == ((e + 1) << 32) | 3 and got.flags[1][me] == ((e + 1) << 32) | 4


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("forced", [False, True])
@pytest.mark.parametrize("reporter", [0, 1, 2])
def test_nonfinite_count_from_one_rank(reporter, forced, dtype):
    """One rank counts non-finite elements in its y1: every rank gets a NaN ratio and the world-1 block's outcome -- a
    reject (then dt underflows), or with min_step forcing the accept, TDQ_RUN_NONFINITE."""
    R, n_seg = 3, 4
    opts, dt = (dict(min_step=0.05), 0.01) if forced else ({}, 0.02)
    counts, ks = _case(n_seg, "accept")
    bad = [0.0] * R
    bad[reporter] = 1.0
    parts = _partials(R, ks, bad)
    cnt = _dev(counts, torch.int64)
    ref = _engine("dopri5", dtype, 16, dt, **opts)[0]
    want_mb = _reference(ref, _dev(_rank_order_sum(parts)), cnt, n_seg)
    m = ref.mbox_host.contents
    assert m.ratio != m.ratio
    assert (m.accept, m.status) == ((1, _lib.RUN_NONFINITE) if forced else (0, _lib.RUN_DT_UNDERFLOW))
    for me in range(R):
        eng = _engine("dopri5", dtype, 16, dt, **opts)[0]
        bufs = _buffers(R)
        _arm(eng, bufs, me, 1)
        _deliver(bufs, me, 1, 0, parts)
        before = _launch(eng, bufs, me, 1, _dev(parts[me]), cnt, n_seg)
        assert bytes(eng.mbox_host.contents) == want_mb, me
        _assert_images(bufs, _expect_send(before, me, 1, 0, parts[me]), me)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_no_exchange_world_one(dtype):
    """A block armed with world 1 decides on its own sums, exactly as an unarmed one, and writes nothing."""
    counts, ks = _case(4, "accept")
    norm_in, cnt = _dev([k * U for k in ks] + [0.0]), _dev(counts, torch.int64)
    ref = _engine("dopri5", dtype, 16, 0.02)[0]
    want_mb = _reference(ref, norm_in, cnt, 4)
    eng = _engine("dopri5", dtype, 16, 0.02)[0]
    bufs = _buffers(1)
    _arm(eng, bufs, 0, 7)
    before = _launch(eng, bufs, 0, 7, norm_in, cnt, 4)
    assert bytes(eng.mbox_host.contents) == want_mb
    _assert_images(bufs, before, "world 1")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_no_exchange_once_halted(dtype):
    """The attempt that ends the solve exchanges; the trailing no-op after it ticks the mailbox and writes nothing, even
    with its flags delivered."""
    R, n_seg, dt, t0, epoch = 2, 1, 0.02, 0.5, 2
    counts, ks = _case(n_seg, "accept")
    parts, cnt = _partials(R, ks), _dev(counts, torch.int64)
    ref = _engine("dopri5", dtype, 16, dt, t0, t_end=t0 + 0.5 * dt)[0]
    eng = _engine("dopri5", dtype, 16, dt, t0, t_end=t0 + 0.5 * dt)[0]
    bufs = _buffers(R)
    _arm(eng, bufs, 0, epoch)
    for seq in range(2):
        _deliver(bufs, 0, epoch, seq, parts)
        before = _launch(eng, bufs, 0, epoch, _dev(parts[0]), cnt, n_seg)
        want_mb = _reference(ref, _dev(_rank_order_sum(parts)), cnt, n_seg)
        assert bytes(eng.mbox_host.contents) == want_mb, seq
        if seq == 0:
            assert eng.mbox_host.contents.done == 1
            _assert_images(bufs, _expect_send(before, 0, epoch, 0, parts[0]), "deciding attempt")
        else:
            _assert_images(bufs, before, "halted")
    assert eng.mbox_host.contents.seq == 2


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_no_exchange_with_ratio_dev(dtype):
    """A controller given the ratio itself (a custom norm) has nothing to exchange: it decides on that ratio."""
    R, n_seg = 3, 1
    counts, ks = _case(n_seg, "reject")
    parts, cnt = _partials(R, ks), _dev(counts, torch.int64)
    ratio = torch.tensor(0.75, dtype=torch.float64 if dtype == torch.float64 else dtype, device="cuda")
    ref = _engine("dopri5", dtype, 16, 0.02)[0]
    want_mb = _reference(ref, _dev(parts[1]), cnt, n_seg, ratio)
    assert ref.mbox_host.contents.accept == 1
    eng = _engine("dopri5", dtype, 16, 0.02)[0]
    bufs = _buffers(R)
    _arm(eng, bufs, 1, 4)
    _deliver(bufs, 1, 4, 0, parts)
    before = _launch(eng, bufs, 1, 4, _dev(parts[1]), cnt, n_seg, ratio)
    assert bytes(eng.mbox_host.contents) == want_mb
    _assert_images(bufs, before, "ratio_dev")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("R,n_seg", [(2, 65), (16, 65), (2, 200)])
def test_too_many_segments_halts(R, n_seg, dtype):
    """An armed block with more segments than the buffers carry halts with TDQ_RUN_EXCHANGE_SEGMENTS instead of deciding
    on its local sums: the mailbox ticks with that status, no buffer is written, and the engine raises the error that
    names the limit.  The same sums on an unarmed block are decided as usual."""
    counts, ks = _case(n_seg, "accept")
    parts, cnt = _partials(R, ks), _dev(counts, torch.int64)
    ref = _engine("dopri5", dtype, 16, 0.02)[0]
    _reference(ref, _dev(_rank_order_sum(parts)), cnt, n_seg)
    m = ref.mbox_host.contents
    assert (m.status, m.accept, m.seq) == (_lib.RUN_OK, 1, 1)
    eng = _engine("dopri5", dtype, 16, 0.02)[0]
    bufs = _buffers(R)
    _arm(eng, bufs, 0, 9)
    _deliver(bufs, 0, 9, 0, parts)
    before = _launch(eng, bufs, 0, 9, _dev(parts[0]), cnt, n_seg)
    mb = eng.mbox_host.contents
    assert (mb.status, mb.accept, mb.n_accept, mb.n_reject, mb.seq) == (_lib.RUN_EXCHANGE_SEGMENTS, 0, 0, 0, 1)
    _assert_images(bufs, before, "too many segments")
    with pytest.raises(_lib.TdqError, match="at most 64 norm segments"):
        eng._raise_if_failed(mb)


# ---- two processes over CUDA IPC ----------------------------------------------------------------------------------------

class _Raw:
    """A device allocation the library made, presented to torch without a copy."""

    def __init__(self, ptr):
        self.__cuda_array_interface__ = {"shape": (NB,), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


def _ipc_case():
    counts, ks = _case(4, "accept")
    return dict(dtype="float64", t_sign=-1.0, dt=0.02, epoch=7, counts=counts, parts=_partials(2, ks))


def _child(arg):
    """Rank 1: open rank 0's buffer, take rank 0's delivery into its own buffer, run one controller whose store lands in
    rank 0's buffer, report the mailbox, close the handle."""
    a = json.loads(arg)
    lib = _lib.load()
    h = _lib.IpcHandle()
    C.memmove(h.bytes, bytes.fromhex(a["handle"]), 64)
    peer = C.c_void_p()
    if lib.tdq_xchg_open(C.byref(h), C.byref(peer)) != 0:
        print("IPC-REFUSED " + lib.tdq_last_error().decode())
        return 3
    dtype = getattr(torch, a["dtype"])
    eng = _engine("dopri5", dtype, 16, a["dt"], 0.5, a["t_sign"])[0]
    bufs = [torch.as_tensor(_Raw(peer.value), device="cuda"), torch.full((NB,), SENT, dtype=torch.uint8, device="cuda")]
    _arm(eng, bufs, 1, a["epoch"])
    x = _image(bufs[1])
    _store(x, a["epoch"], 0, 0, a["parts"][0])
    _upload(bufs[1], x)
    _launch(eng, bufs, 1, a["epoch"], _dev(a["parts"][1]), _dev(a["counts"], torch.int64), len(a["counts"]))
    print("MAILBOX " + bytes(eng.mbox_host.contents).hex())
    del bufs
    _lib.check(lib.tdq_xchg_close(peer))
    return 0


def test_ipc_two_processes():
    """tdq_xchg_create / _open / _close / _destroy and a real cross-process store, still sequential: the child (rank 1)
    runs its controller first, its store lands in the parent's (rank 0's) buffer, then the parent's controller finds the
    flag there.  A scratch buffer stands in for rank 1's buffer on the parent's side.  Both mailboxes equal the world-1
    block's."""
    lib = _lib.load()
    a = _ipc_case()
    own, h = C.c_void_p(), _lib.IpcHandle()
    if lib.tdq_xchg_create(C.byref(own), C.byref(h)) != 0:
        pytest.skip("tdq_xchg_create refused: " + lib.tdq_last_error().decode())
    try:
        mine = torch.as_tensor(_Raw(own.value), device="cuda")
        assert mine.data_ptr() == own.value
        mine.fill_(SENT)
        torch.cuda.synchronize()
        a["handle"] = bytes(h.bytes).hex()
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        env = dict(os.environ, PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests")]))
        p = subprocess.run([sys.executable, os.path.abspath(__file__), json.dumps(a)], capture_output=True, text=True,
                           timeout=180, env=env, cwd=root)
        lines = p.stdout.splitlines()
        if p.returncode == 3 and lines and lines[-1].startswith("IPC-REFUSED"):
            pytest.skip("cudaIpcOpenMemHandle refused: " + lines[-1])
        assert p.returncode == 0, (p.returncode, p.stdout[-2000:], p.stderr[-4000:])
        child_mb = bytes.fromhex(next(l for l in lines if l.startswith("MAILBOX ")).split()[1])

        dtype, epoch, counts, parts = getattr(torch, a["dtype"]), a["epoch"], a["counts"], a["parts"]
        cnt, n_seg = _dev(counts, torch.int64), len(counts)
        got = _image(mine)                                            # the child's store, through CUDA IPC
        assert got.flags[_slot(epoch, 0)][1] == _flag(epoch, 0)
        assert list(got.vals[_slot(epoch, 0)][1][:n_seg + 1]) == parts[1]
        eng = _engine("dopri5", dtype, 16, a["dt"], 0.5, a["t_sign"])[0]
        bufs = [mine, torch.full((NB,), SENT, dtype=torch.uint8, device="cuda")]
        _arm(eng, bufs, 0, epoch)
        before = _launch(eng, bufs, 0, epoch, _dev(parts[0]), cnt, n_seg)
        ref = _engine("dopri5", dtype, 16, a["dt"], 0.5, a["t_sign"])[0]
        want_mb = _reference(ref, _dev(_rank_order_sum(parts)), cnt, n_seg)
        assert child_mb == want_mb
        assert bytes(eng.mbox_host.contents) == want_mb
        _assert_images(bufs, _expect_send(before, 0, epoch, 0, parts[0]), "parent")
        del bufs, mine
        torch.cuda.synchronize()
    finally:
        _lib.check(lib.tdq_xchg_destroy(own))


if __name__ == "__main__":
    sys.exit(_child(sys.argv[1]))
