"""Row compaction of independent-row solves (options={'independent_rows': True, 'compact_rows': True}): the batch sizes
func is called with, and active_rows(), through which func learns which rows it sees."""
import contextlib
import threading

_state = threading.local()


def active_rows():
    """The original row indices of the rows the current func / event_fn call sees, inside a solve with
    options['compact_rows']: an int64 device tensor [B'] in ascending order, whose first entries are the rows still
    running and whose trailing entries repeat the last of them (their results are discarded).  Before the first
    compaction it is arange(B).  None outside such a solve and in the event bisection, which evaluates the whole batch.

    A func that carries per-row data picks its rows with it, e.g. `idx = active_rows(); r = rate if idx is None else
    rate[idx]`.  The tensor is an engine buffer per batch size whose contents change between calls: index with it inside
    the call (a captured graph that does so stays valid on replay), but do not keep it across calls."""
    return getattr(_state, "idx", None)


@contextlib.contextmanager
def rows(idx):
    """active_rows() returns `idx` inside the block."""
    prev = getattr(_state, "idx", None)
    _state.idx = idx
    try:
        yield
    finally:
        _state.idx = prev


def bucket_sizes(B):
    """The batch sizes of a compacting solve of B rows: B_k = ceil(B / 2^k), k = 0, 1, ... down to 1, each once
    (ceil(log2 B) + 1 sizes)."""
    sizes = [int(B)]
    while sizes[-1] > 1:
        sizes.append((sizes[-1] + 1) // 2)          # ceil(ceil(B / 2^k) / 2) = ceil(B / 2^(k+1))
    return sizes


def pick(sizes, n_running):
    """(size, threshold) for n_running rows: the smallest size that holds them, and the running count at or below which
    the solve pauses for the next compaction (the next smaller size; 0 at the smallest, where it never pauses)."""
    j = max(i for i, s in enumerate(sizes) if s >= n_running) if n_running > 0 else len(sizes) - 1
    return sizes[j], (sizes[j + 1] if j + 1 < len(sizes) else 0)
