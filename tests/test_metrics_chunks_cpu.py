"""CPU tests (no GPU): the chunking that sequence_metrics, official_sequence_metrics and LPIPS share -- the chunk walk
(_chunks), the chunk-length search and its refusal (_chunk_len) -- against the loops each entry point ran on its own
before they shared them, written out here as the specification, and the refusal text each entry point reports."""
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                            # noqa: E402

M = T.metrics


# ---- the specification: each entry point's own loops -----------------------------------------------------------------

def spec_walk(total, n, overlap):
    """sequence_metrics' and official_sequence_metrics' walk; the first `first` frames of a chunk were scored by the
    chunk before"""
    out, s = [], 0
    while True:
        e = min(s + n, total)
        out.append((s, e, 1 if s > 0 and overlap else 0))
        if e == total:
            break
        s = e - 1 if overlap else e
    return out


def spec_lpips_walk(total, n):
    """LPIPS.__call__'s walk"""
    return [(s, min(s + n, total), 0) for s in range(0, total, n)]


def spec_lpips_len(N, chunk_bytes, budget, h, w):
    n = N
    while n > 1 and chunk_bytes(n) > budget:
        n -= 1
    if chunk_bytes(n) > budget:
        raise ValueError(f'max_workspace_bytes={budget} is below the {chunk_bytes(1)} bytes that one '
                         f'pair of {h}x{w} frames needs')
    return n


def spec_sequence_len(T_, tof, chunk_bytes, budget, h, w):
    n, n_min = T_, (2 if tof and T_ >= 2 else 1)
    while n > n_min and chunk_bytes(n) > budget:
        n -= 1
    if chunk_bytes(n) > budget:
        raise ValueError(f'max_workspace_bytes={budget} is below the {chunk_bytes(n)} bytes that '
                         f'{n} frames of {h}x{w} need')
    return n


def spec_official_len(n_s, overlap, chunk_bytes, budget, h, w):
    n, n_min = n_s, min(n_s, 2 if overlap else 1)
    while n > n_min and chunk_bytes(n) > budget:
        n -= 1
    if chunk_bytes(n) > budget:
        raise ValueError(f'max_workspace_bytes={budget} is below the {chunk_bytes(n)} bytes that '
                         f'{n} frames of {h}x{w} need')
    return n


# ---- the shared walk -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('overlap', [False, True])
def test_chunks_follow_the_loops(overlap):
    for total in range(1, 10):
        for n in range(2 if overlap else 1, 10):
            got = list(M._chunks(total, n, overlap))
            assert got == spec_walk(total, n, overlap), (total, n)
            if not overlap:
                assert got == spec_lpips_walk(total, n), (total, n)
            assert all(0 < e - s <= n for s, e, _ in got)
            # every frame's own result is kept once, in order; with overlap so is every consecutive pair
            assert [i for s, e, first in got for i in range(s + first, e)] == list(range(total))
            if overlap:
                assert [i for s, e, _ in got for i in range(s + 1, e)] == list(range(1, total))


def test_chunks_pinned():
    assert list(M._chunks(5, 2, True)) == [(0, 2, 0), (1, 3, 1), (2, 4, 1), (3, 5, 1)]
    assert list(M._chunks(7, 3, True)) == [(0, 3, 0), (2, 5, 1), (4, 7, 1)]
    assert list(M._chunks(7, 3, False)) == [(0, 3, 0), (3, 6, 0), (6, 7, 0)]
    assert list(M._chunks(4, 9, True)) == [(0, 4, 0)]
    assert list(M._chunks(1, 1, True)) == [(0, 1, 0)]          # one frame: one chunk, nothing to overlap


def test_chunks_refuse_a_walk_that_never_ends():
    for total in (2, 5, 9):
        with pytest.raises(ValueError, match='never cover'):
            list(M._chunks(total, 1, True))                    # each chunk would start where the last one did
        with pytest.raises(ValueError, match='never cover'):
            list(M._chunks(total, 0, False))


# ---- the shared chunk-length search ----------------------------------------------------------------------------------

H, W = 24, 40
CHUNK_BYTES = (
    lambda n: 1000 + 300 * n,                                  # frames and features: linear
    lambda n: 500 * n + (800 * (n - 1) if n >= 2 else 0),      # plus flows between consecutive frames
)
BUDGETS = range(0, 5000, 97)


def _outcome(fn):
    try:
        return fn()
    except ValueError as e:
        return str(e)


def _frames_need(chunk_bytes):
    return lambda n: f'{chunk_bytes(n)} bytes that {n} frames of {H}x{W} need'


def test_chunk_len_as_lpips_call():
    for cb in CHUNK_BYTES:
        for N in range(1, 10):
            for b in BUDGETS:
                got = _outcome(lambda: M._chunk_len(N, 1, cb, b, lambda n: f'{cb(1)} bytes that one pair of '
                                                                           f'{H}x{W} frames needs'))
                assert got == _outcome(lambda: spec_lpips_len(N, cb, b, H, W)), (N, b)


def test_chunk_len_as_sequence_metrics():
    for cb in CHUNK_BYTES:
        for tof in (False, True):
            for T_ in range(1, 10):
                for b in BUDGETS:
                    got = _outcome(lambda: M._chunk_len(T_, 2 if tof and T_ >= 2 else 1, cb, b, _frames_need(cb)))
                    assert got == _outcome(lambda: spec_sequence_len(T_, tof, cb, b, H, W)), (tof, T_, b)


def test_chunk_len_as_official_sequence_metrics():
    for cb in CHUNK_BYTES:
        for overlap in (False, True):
            for n_s in range(1, 10):
                for b in BUDGETS:
                    got = _outcome(lambda: M._chunk_len(n_s, min(n_s, 2 if overlap else 1), cb, b, _frames_need(cb)))
                    assert got == _outcome(lambda: spec_official_len(n_s, overlap, cb, b, H, W)), (overlap, n_s, b)


def test_chunk_len_pinned():
    cb = CHUNK_BYTES[1]                                        # 500, 1800, 3100, 4400, ... bytes for 1, 2, 3, 4 frames
    assert M._chunk_len(4, 2, cb, 5000, _frames_need(cb)) == 4
    assert M._chunk_len(4, 2, cb, 4399, _frames_need(cb)) == 3
    assert M._chunk_len(4, 2, cb, 1800, _frames_need(cb)) == 2
    with pytest.raises(ValueError) as e:
        M._chunk_len(4, 2, cb, 1799, _frames_need(cb))
    assert str(e.value) == 'max_workspace_bytes=1799 is below the 1800 bytes that 2 frames of 24x40 need'


# ---- what each entry point reports -----------------------------------------------------------------------------------

def test_entry_points_name_their_smallest_chunk():
    """the refusal of a 1-byte budget names the bytes of the smallest chunk (callers parse them) and its frames: two
    with a temporal metric, else one.  It comes before any device work."""
    lp = M.LPIPS.__new__(M.LPIPS)
    lp.device = torch.device('cuda', 0)
    x = np.zeros((6, 64, 64, 3), np.uint8)                    # official: cutfr = 2 leaves 2 scored frames
    cases = (
        (lambda b: M.sequence_metrics(x, x, lpips=lp, max_workspace_bytes=b), 'that 2 frames of 64x64 need'),
        (lambda b: M.sequence_metrics(x, x, tof=False, lpips=lp, max_workspace_bytes=b), 'that 1 frames of 64x64 need'),
        (lambda b: M.official_sequence_metrics(x, x, keys=('LPIPS', 'tLP100'), lpips=lp, max_workspace_bytes=b),
         'that 2 frames of 64x64 need'),
        (lambda b: M.official_sequence_metrics(x, x, keys=('LPIPS',), lpips=lp, max_workspace_bytes=b),
         'that 1 frames of 64x64 need'),
        (lambda b: lp(x, x, max_workspace_bytes=b), 'that one pair of 64x64 frames needs'),
    )
    for fn, tail in cases:
        with pytest.raises(ValueError) as e:
            fn(1)
        assert re.fullmatch(r'max_workspace_bytes=1 is below the \d+ bytes ' + tail, str(e.value)), str(e.value)
