"""Batch sizes at which the whole-attempt kernels (csrc/tdq_attempt.cu) run several 32-row tiles in one CTA.

k_linear_attempt, k_linear_rows_attempt and k_linear_solve launch min(ceil(B / 32), P) CTAs, P the device's SM count
(tdq_grid with one block per SM), and CTA c runs tiles c, c + P, c + 2P, ...  A CTA therefore takes a second tile once
ceil(B / 32) > P.  Sizes are written in terms of P ("32P+1") so that test ids do not depend on the card; `rows` turns
them into row counts for the device the tests run on."""
import ctypes as C

TILE = 32


def sm_count():
    """P: the SM count the library's grid rule reads (tdq_device_sm_count)."""
    from torchdiffeq_b200 import _lib
    n = C.c_int()
    _lib.check(_lib.load().tdq_device_sm_count(C.byref(n)))
    return n.value


def rows(size, P):
    """size: an int, or "aP", "aP+b" (a 32-row tiles per SM plus b rows)."""
    if isinstance(size, int):
        return size
    a, _, b = size.partition("P")
    return int(a) * P + (int(b) if b else 0)


def tiles(B):
    return -(-B // TILE)


def multi_tile(B, P):
    """at least one CTA runs two or more tiles"""
    return tiles(B) > P
