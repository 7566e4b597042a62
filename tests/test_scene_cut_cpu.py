"""CPU tests (no GPU): the scene-cut specification oracle/scene_cut.py -- the 8-bit codes, the decision rules on
hand-made mafd sequences, a SAD above 2**32 -- and the argument checks of FRNet.stream(scene_cut=) and
tg_scene_cut, which reject bad values with ValueError and the documented codes before any device work."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import scene_cut as S              # noqa: E402

L = sys.modules['tecogan-pytorch_b200.lib']
ops = sys.modules['tecogan-pytorch_b200.ops']
P = ctypes.c_void_p(16)                        # a non-null, aligned pointer that is never dereferenced
INVALID, UNSUPPORTED = -1, -2


def test_codes_of_decoded_uint8_are_the_bytes():
    v = np.arange(256)
    assert np.array_equal(S.q(v.astype(np.float32) / np.float32(255)), v)
    # round half to even on the fp32 product, clamp, NaN as 0
    assert list(S.q(np.float32([0.5 / 255, 1.5 / 255, -0.5, 1.5, np.nan, np.inf, -np.inf]))) == [0, 2, 0, 255, 0,
                                                                                                  255, 0]


def _run(mafds, resets=(), threshold=10.0):
    """decide() over a sequence of mafd values; frame 0 is the stream's start (a reset)."""
    pm, out = -1.0, []
    for i, m in enumerate(mafds):
        score, cut, pm = S.decide(m, pm, i == 0 or i in resets, threshold)
        out.append((score, cut, pm))
    return out


def test_first_frame_and_frame_after_a_restart_score_zero():
    r = _run([50.0, 2.0, 2.5, 40.0, 41.0, 1.0])
    assert [s for s, _, _ in r] == [0.0, 0.0, 0.5, 37.5, 0.0, 1.0]
    assert [c for _, c, _ in r] == [False, False, False, True, False, False]
    # after the cut the state is -1, so frame 4 only records its mafd; frame 5 drops by 40 but its own mafd is 1
    assert [pm for _, _, pm in r] == [-1.0, 2.0, 2.5, -1.0, 41.0, 1.0]


def test_score_is_the_smaller_of_mafd_and_its_change():
    r = _run([0.0, 30.0, 30.5, 5.0, 4.0], threshold=100.0)
    assert [s for s, _, _ in r] == [0.0, 0.0, 0.5, 5.0, 1.0]
    assert not any(c for _, c, _ in r)


def test_threshold_is_inclusive():
    r = _run([0.0, 1.0, 11.0], threshold=10.0)
    assert r[2] == (10.0, True, -1.0)
    r = _run([0.0, 1.0, 10.999], threshold=10.0)
    assert r[2][1] is False and r[2][0] < 10.0
    assert S.decide(100.0, 0.0, False, 100.0) == (100.0, True, -1.0)


def test_caller_reset_overrides_a_cut():
    r = _run([0.0, 1.0, 60.0, 61.0], resets={2})
    assert r[2] == (0.0, False, -1.0)
    assert r[3] == (0.0, False, 61.0)


def test_sad_above_2_pow_32():
    a = np.ones((1, 4105, 4105), np.float32)
    b = np.zeros_like(a)
    sad = S.sad(a, b)
    assert sad == 255 * 4105 * 4105 and sad > 2 ** 32
    assert S.mafd_of(sad, a.size) == 100.0
    assert S.mafd_of(2 ** 40 + 1, 3 * 2400 * 2400) == float(np.float64(2 ** 40 + 1) * 100.0 / (3 * 2400 * 2400) / 255.0)


def test_step_and_stream_agree():
    rng = np.random.default_rng(3)
    lr = rng.uniform(-0.5, 1.5, (6, 3, 5, 7)).astype(np.float32)
    scores, cuts = S.stream(lr, {4}, 1.0)
    pm, prev = np.array([-1.0]), np.zeros_like(lr[:1])
    for i in range(6):
        reset = i in (0, 4)
        if reset:
            prev = np.zeros_like(lr[:1])
        s, c, pm = S.step(lr[i:i + 1], prev, pm, [reset], 1.0)
        assert s[0] == scores[i] and c[0] == cuts[i]
        prev = lr[i:i + 1]


def test_two_synthetic_shots_give_one_cut():
    """At 1 px/frame the joint of two seeded clips is the only frame at or above 10."""
    a = synthetic.make_clip(1, 8, 3, 134, 320).numpy()
    b = synthetic.make_clip(2, 8, 3, 134, 320).numpy()
    scores, cuts = S.stream(np.concatenate([a, b]), set(), 10.0)
    assert list(np.nonzero(cuts)[0]) == [8]
    assert scores[8] > 15.0 and np.delete(scores, 8).max() < 0.1


# ---------------------------------------------------------------------------- FRNet.stream(scene_cut=)
def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


@pytest.mark.parametrize('value', [True, False, '10', b'10', [10.0], (10.0,), complex(10, 0), float('nan'),
                                   float('inf'), -float('inf'), 0, 0.0, -1.0, 100.0001, 1e9, np.float64(np.nan),
                                   np.float32(0)])
def test_stream_refuses_bad_scene_cut(value):
    with pytest.raises(ValueError):
        _net().stream(2, 16, 24, device='cuda', scene_cut=value)


def test_stream_accepts_scene_cut():
    net = _net()
    for value in (10, 10.0, 100, 1e-6, np.float32(25.5), np.int64(3)):
        s = net.stream(2, 16, 24, device='cuda', scene_cut=value)
        assert type(s.scene_cut) is float and s.scene_cut == float(value)
        assert s.last_cuts is None and s.last_scores is None
    for kw in (dict(input='nv12', out_format='p010'), dict(input='float32'), dict(out_size=(48, 72))):
        assert net.stream(2, 16, 24, device='cuda', scene_cut=10.0, **kw).scene_cut == 10.0
    s = net.stream(2, 16, 24, device='cuda')
    assert s.scene_cut is None and s.last_cuts is None and s.last_scores is None


# ---------------------------------------------------------------------------- tg_scene_cut argument checks
def _call(a=P, b=P, n=2, c=3, h=8, w=8, reset=P, thr=10.0, pm=P, work=P, score=P, cut=P):
    return L.load().tg_scene_cut(a, b, n, c, h, w, reset, thr, pm, work, score, cut, None)


def _err():
    return L.load().tg_last_error_string()


def test_scene_cut_rejects_bad_arguments_without_a_gpu():
    for kw in (dict(a=None), dict(b=None), dict(pm=None), dict(work=None), dict(score=None), dict(cut=None)):
        assert _call(**kw) == INVALID
        assert b'null' in _err()
    for kw in (dict(n=0), dict(c=0), dict(h=-1), dict(w=0)):
        assert _call(**kw) == INVALID
        assert b'bad size' in _err()
    for kw in (dict(a=ctypes.c_void_p(18)), dict(b=ctypes.c_void_p(17)), dict(reset=ctypes.c_void_p(18)),
               dict(cut=ctypes.c_void_p(19)), dict(pm=ctypes.c_void_p(20)), dict(work=ctypes.c_void_p(12)),
               dict(score=ctypes.c_void_p(4))):
        assert _call(**kw) == INVALID
        assert b'aligned' in _err()
    for thr in (0.0, -1.0, 100.5, math.nan, math.inf, -math.inf, 1e300):
        assert _call(thr=thr) == INVALID
        assert b'threshold' in _err()
    assert _call(c=5) == UNSUPPORTED
    assert b'channels' in _err()
    assert _call(n=(1 << 23) + 1, c=1, h=1024, w=1024) == UNSUPPORTED      # 256 CTAs per slot
    assert b'grid' in _err()


def test_ops_wrapper_refuses_before_device_work():
    assert L.SCENE_CUT_WORK_BYTES == 16
    assert ops.scene_cut_threshold_ok(100.0) and not ops.scene_cut_threshold_ok(0.0)
    x = torch.zeros(2, 3, 8, 8)
    with pytest.raises(T.TecoganB200Error, match='CUDA'):
        ops.scene_cut(x, x, None, 10.0, torch.zeros(2, dtype=torch.float64), torch.zeros(4, dtype=torch.int64),
                      torch.zeros(2, dtype=torch.float64), torch.zeros(2, dtype=torch.int32))
