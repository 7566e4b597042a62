"""Scene-cut detection of streamed video, restated in integer / float64 numpy.

This is the specification of tg_scene_cut (FRNet.stream(scene_cut=threshold)).  For each slot, at each step, a is
the step's current LR frame and b its previous one (fp32 [c,h,w], as the step sees them: decoded on the device, and
zeroed by a caller reset of this step):

  q(x)   = clip(rint(float32(x) * float32(255)), 0, 255)   fp32 product, round half to even, as integers; NaN -> 0
  SAD    = sum |q(a) - q(b)|                               exact integer (may exceed 2**32)
  mafd   = float64(SAD) * 100.0 / count / 255.0            float64, in that order; count = c*h*w

For uint8 input q gives back the input bytes (the decode is float32(v) / float32(255)).  Each slot keeps the
previous mafd pm, -1 meaning none:

  caller reset at this step (or the stream's first push):  score 0, cut False, pm := -1
  otherwise, pm < 0:                                        score 0, cut False, pm := mafd
  otherwise:  score = min(max(min(mafd, |mafd - pm|), 0), 100), cut = score >= threshold,
              pm := -1 if cut else mafd

The score min(mafd, |delta mafd|) is the one of ffmpeg's scdet filter: steady high motion keeps |delta mafd| small and
a jump raises both.  The restart rule (pm := -1 after any restart, detected or requested) differs from scdet, which
starts from pm = 0 and so flags the second frame of every video, and which flags the frame after a cut a second time
(the cut raised mafd, the next frame lowers it again).  The numbers are therefore not scdet's.
"""
import numpy as np


def q(x):
    """8-bit codes of fp32 frames: clip(rint(x * 255), 0, 255) with an fp32 product, as int16 (room for the
    difference of two codes); NaN counts as 0."""
    v = np.rint(np.asarray(x, dtype=np.float32) * np.float32(255))
    return np.clip(np.nan_to_num(v, nan=0.0), 0, 255).astype(np.int16)


def sad(a, b):
    """Exact integer sum of |q(a) - q(b)| (a Python int; summed in int64)."""
    return int(np.abs(q(a) - q(b)).sum(dtype=np.int64))


def mafd_of(sad_value, count):
    """float64(SAD) * 100.0 / count / 255.0, in that order."""
    return float(np.float64(sad_value) * 100.0 / float(count) / 255.0)


def decide(mafd, pm, reset, threshold):
    """One step of one slot: (score, cut, new pm) from its mafd, its state pm and the caller's reset flag."""
    if reset:
        return 0.0, False, -1.0
    if pm < 0:
        return 0.0, False, mafd
    score = min(max(min(mafd, abs(mafd - pm)), 0.0), 100.0)
    cut = score >= threshold
    return score, cut, (-1.0 if cut else mafd)


def step(a, b, pm, reset, threshold):
    """One launch over n slots: a, b [n,c,h,w] fp32 (current, previous), pm float64 [n], reset bools [n] ->
    (score float64 [n], cut bool [n], new pm float64 [n])."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    n = a.shape[0]
    count = int(np.prod(a.shape[1:]))
    score, cut, new = np.zeros(n), np.zeros(n, bool), np.zeros(n)
    for k in range(n):
        m = mafd_of(sad(a[k], b[k]), count)
        score[k], cut[k], new[k] = decide(m, float(pm[k]), bool(reset[k]), threshold)
    return score, cut, new


def stream(lr, resets, threshold):
    """A stream of one slot's LR frames lr [t,c,h,w] (fp32, as decoded) with caller resets at the frame indices in
    `resets` (frame 0 is always a restart) -> (score float64 [t], cut bool [t]).  The step's previous frame is the
    previous decoded frame, or zeros after a restart (the reset zeroes it before the score is taken)."""
    lr = np.asarray(lr, np.float32)
    t = lr.shape[0]
    count = int(np.prod(lr.shape[1:]))
    scores, cuts = np.zeros(t), np.zeros(t, bool)
    pm, prev = -1.0, np.zeros_like(lr[0])
    for i in range(t):
        reset = i == 0 or i in resets
        if reset:
            prev = np.zeros_like(lr[0])
        m = mafd_of(sad(lr[i], prev), count)
        scores[i], cuts[i], pm = decide(m, pm, reset, threshold)
        prev = lr[i]
    return scores, cuts
