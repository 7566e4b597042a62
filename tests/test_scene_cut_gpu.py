"""pytest -m gpu: scene-cut detection of streamed video, FRNet.stream(scene_cut=threshold).

The kernel tg_scene_cut is checked bit for bit against oracle/scene_cut.py (score as float64 bits, cut, and the
per-slot state prev_mafd) on ragged, misaligned and guard-banded buffers.  End to end, a stream with scene_cut on a
slot whose video changes shot at frame 8 gives the bytes of a stream without it that the caller restarts there with
reset=, whatever the chunking of the pushes, and reports the cut (last_cuts / last_scores) as the oracle does on the
decoded LR frames."""
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
from oracle import yuv_color as C              # noqa: E402

pytestmark = pytest.mark.gpu

L = sys.modules['tecogan-pytorch_b200.lib']
ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
G = 8                                          # guard words on each side of every output
SENT_F64, SENT_I32 = -12345.5, -777
BD4 = dict(scale=4, degradation='BD', h=134, w=320, out_size=(402, 960))
BI2 = dict(scale=2, degradation='BI', h=36, w=52, out_size=(54, 130))
THR = 10.0


# ---------------------------------------------------------------------------- kernel against the oracle
class Launcher:
    """tg_scene_cut on n slots with prev_mafd / score / cut / work inside guard bands."""

    def __init__(self, n):
        self.n = n
        self.pm_buf = torch.full((n + 2 * G,), SENT_F64, dtype=torch.float64, device=DEV)
        self.score_buf = torch.full((n + 2 * G,), SENT_F64, dtype=torch.float64, device=DEV)
        self.cut_buf = torch.full((n + 2 * G,), SENT_I32, dtype=torch.int32, device=DEV)
        self.work_buf = torch.full((2 * n + 2 * G,), -1, dtype=torch.int64, device=DEV)
        self.pm, self.score, self.cut = self.pm_buf[G:G + n], self.score_buf[G:G + n], self.cut_buf[G:G + n]
        self.work = self.work_buf[G:G + 2 * n]
        self.pm.fill_(-1.0)
        self.work.zero_()

    def __call__(self, a, b, reset, thr=THR):
        r = None if reset is None else torch.tensor(np.asarray(reset, np.int32), device=DEV)
        ops.scene_cut(a, b, r, thr, self.pm, self.work, self.score, self.cut)
        torch.cuda.synchronize()
        self.check_guards()
        return (self.score.cpu().numpy().copy(), self.cut.cpu().numpy().copy(), self.pm.cpu().numpy().copy())

    def check_guards(self):
        assert (self.pm_buf[:G] == SENT_F64).all() and (self.pm_buf[G + self.n:] == SENT_F64).all()
        assert (self.score_buf[:G] == SENT_F64).all() and (self.score_buf[G + self.n:] == SENT_F64).all()
        assert (self.cut_buf[:G] == SENT_I32).all() and (self.cut_buf[G + self.n:] == SENT_I32).all()
        assert (self.work_buf[:G] == -1).all() and (self.work_buf[G + 2 * self.n:] == -1).all()
        assert (self.work == 0).all(), 'the workspace must be left zeroed'


def _placed(x, offset, fill):
    """x [n,c,h,w] fp32 on the device at `offset` floats past a 256-byte-aligned start, `fill` around it (the two
    frames get fills of codes 255 and 0, so a read outside them would add to the SAD)."""
    flat = torch.full((x.size + offset + 64,), fill, device=DEV)
    v = flat[offset:offset + x.size].view(x.shape)
    v.copy_(torch.from_numpy(x))
    return v


def _same_bits(got, want):
    score, cut, pm = got
    ws, wc, wp = want
    assert np.array_equal(score.view(np.int64), np.asarray(ws, np.float64).view(np.int64)), (score, ws)
    assert np.array_equal(cut != 0, wc), (cut, wc)
    assert np.array_equal(pm.view(np.int64), np.asarray(wp, np.float64).view(np.int64)), (pm, wp)


@pytest.mark.parametrize('n,c,h,w', [(1, 1, 1, 1), (2, 3, 1, 1), (3, 1, 7, 5), (5, 3, 3, 7), (4, 3, 17, 33),
                                     (2, 3, 134, 320), (1, 1, 129, 257), (5, 1, 64, 64)])
@pytest.mark.parametrize('offsets', [(0, 0), (1, 1), (3, 1)], ids=['aligned', 'same_offset', 'mixed_offset'])
def test_kernel_matches_oracle_bit_for_bit(n, c, h, w, offsets):
    """A sequence of 12 launches per slot: frames that alternate between a near copy of the previous one and an
    unrelated one, so both restart rules (pm < 0 after a restart, pm := -1 after a cut) and the threshold are crossed;
    random caller resets; values in [-0.5, 1.5] so the clamp of q is exercised."""
    rng = np.random.default_rng(n * 1000 + c * 100 + h + w)
    launch = Launcher(n)
    pm = np.full(n, -1.0)
    seen_cut = False
    prev = rng.uniform(-0.5, 1.5, (n, c, h, w)).astype(np.float32)
    for step in range(12):
        far = (step + np.arange(n)) % 4 == 2                # every slot jumps to an unrelated frame every 4 steps
        cur = np.where(far[:, None, None, None], rng.uniform(-0.5, 1.5, (n, c, h, w)),
                       prev + rng.normal(0, 0.01, (n, c, h, w))).astype(np.float32)
        reset = [step == 0 or bool(rng.random() < 0.15) for _ in range(n)]
        reset_arg = None if step == 5 else reset          # one launch with no mask at all
        if reset_arg is None:
            reset = [False] * n
        a, b = _placed(cur, offsets[0], 3.0), _placed(prev, offsets[1], -3.0)
        want = S.step(cur, prev, pm, reset, THR)
        got = launch(a, b, reset_arg)
        _same_bits(got, want)
        pm = want[2]
        seen_cut |= bool(want[1].any())
        prev = cur
    assert seen_cut or h * w * c < 4                     # a 1-3 value frame may never cross the threshold


def test_two_launches_give_identical_bits():
    rng = np.random.default_rng(7)
    n, c, h, w = 3, 3, 67, 91
    x = [_placed(rng.uniform(-0.5, 1.5, (n, c, h, w)).astype(np.float32), 1, f) for f in (3.0, -3.0)]
    launch = Launcher(n)
    launch(x[0], x[1], [0, 0, 0])                        # pm := mafd
    pm0 = launch.pm.clone()
    first = launch(x[1], x[0], [0, 1, 0])
    launch.pm.copy_(pm0)
    second = launch(x[1], x[0], [0, 1, 0])
    for f, s in zip(first, second):
        assert np.array_equal(f.view(np.uint8), s.view(np.uint8))


def test_sad_above_2_pow_32():
    """One slot of 3x2400x2400: a frame of ones against zeros (SAD = 255 * 17.28e6 > 2**32), then a frame of mostly
    saturated codes against zeros, scored against the first."""
    n, c, h, w = 1, 3, 2400, 2400
    rng = np.random.default_rng(11)
    launch = Launcher(n)
    ones = torch.ones(n, c, h, w, device=DEV)
    zeros = torch.zeros(n, c, h, w, device=DEV)
    bright = rng.uniform(0.9, 2.0, (n, c, h, w)).astype(np.float32)
    assert S.sad(bright, np.zeros_like(bright)) > 2 ** 32
    pm = np.full(n, -1.0)
    for a_np, a in ((np.ones((n, c, h, w), np.float32), ones), (bright, torch.from_numpy(bright).to(DEV))):
        want = S.step(a_np, np.zeros_like(a_np), pm, [False], THR)
        _same_bits(launch(a, zeros, [0]), want)
        pm = want[2]
    assert pm[0] != 100.0 and want[0][0] > 0                 # the second launch scored against the first's 100


# ---------------------------------------------------------------------------- streams end to end
def _net(scale, degradation):
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def nets():
    return {'bd4': _net(4, 'BD'), 'bi2': _net(2, 'BI')}


def _two_shot_rgb(h, w):
    """uint8 RGB [2,16,h,w,3]: slot 0 is make_clip(1) then make_clip(2), 8 frames each (a cut at frame 8); slot 1
    one continuous clip.  1 px/frame."""
    s0 = np.concatenate([synthetic.make_clip(1, 8, 3, h, w).numpy(), synthetic.make_clip(2, 8, 3, h, w).numpy()])
    s1 = synthetic.make_clip(3, 16, 3, h, w).numpy()
    clips = np.stack([s0, s1])                                            # [2,16,3,h,w]
    return np.ascontiguousarray(np.rint(clips * 255.0).astype(np.uint8).transpose(0, 1, 3, 4, 2))


# (name, stream kwargs, frames of the uint8 RGB clip, decoded fp32 LR frames [..., h, w, 3] for the oracle)
def _case(name, rgb):
    f255 = lambda v: v.astype(np.float32) / np.float32(255)                # noqa: E731
    if name in ('rgb', 'device', 'out_size'):
        return dict(), rgb, f255(rgb)
    if name == 'bgr':
        return dict(channel_order='bgr'), np.ascontiguousarray(rgb[..., ::-1]), f255(rgb)
    if name == 'nv12':
        yuv = C.rgb_to_yuv(rgb, 'nv12', 'bt601')
        return dict(input='nv12', out_format='nv12'), yuv, f255(C.yuv_to_rgb(yuv, 'nv12', 'bt601'))
    if name == 'p010':
        yuv = C.rgb_to_yuv(np.rint(rgb.astype(np.float64) * (1023.0 / 255.0)).astype(np.int64), 'p010', 'bt709')
        dec = C.yuv_to_rgb(yuv, 'p010', 'bt709').astype(np.float32) / np.float32(1023)
        return dict(input='p010', out_format='p010', in_color='bt709', out_color='bt709'), yuv, dec
    if name == 'float32':
        f = np.ascontiguousarray(f255(rgb).transpose(0, 1, 4, 2, 3))
        return dict(input='float32'), f, f255(rgb)
    raise AssertionError(name)


def _push(stream, frames, chunks, out, resets=None):
    res, cuts, scores, i = [], [], [], 0
    for j, k in enumerate(chunks):
        src = torch.from_numpy(np.ascontiguousarray(frames[:, i:i + k]))
        if out == 'device':
            src = src.to(DEV)
        o = stream.push(src, reset=resets[j] if resets else None, out=out)
        res.append(o.cpu().numpy() if isinstance(o, torch.Tensor) else o)
        if stream.scene_cut is not None:
            lc, ls = stream.last_cuts, stream.last_scores
            if out == 'device':
                assert lc.is_cuda and ls.is_cuda and lc.dtype == torch.bool and ls.dtype == torch.float64
                lc, ls = lc.cpu().numpy(), ls.cpu().numpy()
            else:
                assert isinstance(lc, np.ndarray) and lc.dtype == bool and ls.dtype == np.float64
            assert lc.shape == ls.shape == (stream.n, k)
            cuts.append(lc)
            scores.append(ls)
        i += k
    cat = lambda v: np.concatenate(v, axis=1) if v else None               # noqa: E731
    return cat(res), cat(cuts), cat(scores)


CASES = ['rgb', 'bgr', 'nv12', 'p010', 'float32', 'out_size', 'device']


@pytest.mark.parametrize('geom', [BD4, BI2], ids=['bd4', 'bi2'])
@pytest.mark.parametrize('case', CASES)
def test_detected_cut_equals_explicit_reset(geom, case, nets):
    net = nets['bd4' if geom is BD4 else 'bi2']
    h, w = geom['h'], geom['w']
    kw, frames, decoded = _case(case, _two_shot_rgb(h, w))
    if case == 'out_size':
        kw = dict(out_size=geom['out_size'])
    out = 'device' if case == 'device' else 'host'
    plain = net.stream(2, h, w, device=DEV, **kw)
    want, _, _ = _push(plain, frames, [8, 8], out, resets=[None, [True, False]])
    plain.close()
    # the oracle on the decoded LR frames: slot 0 restarts at its detected cut, slot 1 never
    o_scores, o_cuts = zip(*(S.stream(decoded[k], set(), THR) for k in range(2)))
    o_scores, o_cuts = np.stack(o_scores), np.stack(o_cuts)
    assert list(zip(*np.nonzero(o_cuts))) == [(0, 8)], 'the test clip must have exactly one detectable cut'
    for chunks in ([5, 3, 8], [3, 7, 6]):
        s = net.stream(2, h, w, device=DEV, scene_cut=THR, **kw)
        got, cuts, scores = _push(s, frames, chunks, out)
        s.close()
        assert got.dtype == want.dtype and np.array_equal(got, want), (case, chunks, int((got != want).sum()))
        assert np.array_equal(cuts, o_cuts), (case, chunks, np.nonzero(cuts))
        assert np.array_equal(scores.view(np.int64), o_scores.view(np.int64)), (case, chunks)


@pytest.mark.parametrize('n', [1, 2])
@pytest.mark.parametrize('out', ['device', 'host'])
def test_one_frame_pushes_report_each_frame(n, out, nets):
    """Pushes of one frame each (the per-frame pattern of decoded device surfaces), n = 1 and 2 slots.  Every
    push's last_cuts / last_scores are kept as returned and checked against the oracle only after the last push,
    so a report that shares memory with the stream's buffers (overwritten by the next push) fails."""
    net, h, w = nets['bi2'], BI2['h'], BI2['w']
    rgb = _two_shot_rgb(h, w)[:n]
    plain = net.stream(n, h, w, device=DEV)
    want, _, _ = _push(plain, rgb, [8, 8], out, resets=[None, [True] + [False] * (n - 1)])
    plain.close()
    s = net.stream(n, h, w, device=DEV, scene_cut=THR)
    got, kept = [], []
    for i in range(16):
        src = torch.from_numpy(np.ascontiguousarray(rgb[:, i:i + 1]))
        o = s.push(src.to(DEV) if out == 'device' else src, out=out)
        got.append(o.cpu().numpy() if out == 'device' else o)
        kept.append((s.last_cuts, s.last_scores))
    s.close()
    assert np.array_equal(np.concatenate(got, axis=1), want)
    o_scores, o_cuts = zip(*(S.stream(rgb[k].astype(np.float32) / np.float32(255), set(), THR) for k in range(n)))
    o_scores, o_cuts = np.stack(o_scores), np.stack(o_cuts)
    for i, (lc, ls) in enumerate(kept):
        if out == 'device':
            assert lc.is_cuda and ls.is_cuda
            lc, ls = lc.cpu().numpy(), ls.cpu().numpy()
        assert lc.shape == ls.shape == (n, 1) and lc.dtype == bool and ls.dtype == np.float64
        assert np.array_equal(lc[:, 0], o_cuts[:, i]), i
        assert np.array_equal(ls[:, 0].view(np.int64), o_scores[:, i].view(np.int64)), (i, ls[:, 0], o_scores[:, i])
    assert o_cuts[0, 8] and o_cuts.sum() == 1


def test_caller_reset_on_the_cut_frame(nets):
    net, h, w = nets['bd4'], BD4['h'], BD4['w']
    rgb = _two_shot_rgb(h, w)
    plain = net.stream(2, h, w, device=DEV)
    want, _, _ = _push(plain, rgb, [8, 8], 'host', resets=[None, [True, False]])
    s = net.stream(2, h, w, device=DEV, scene_cut=THR)
    got, cuts, scores = _push(s, rgb, [8, 8], 'host', resets=[None, [True, False]])
    assert np.array_equal(got, want)
    assert not cuts.any() and scores[0, 8] == 0.0 and scores[0, 9] == 0.0
    o_scores, _ = S.stream(rgb[0].astype(np.float32) / np.float32(255), {8}, THR)
    assert np.array_equal(scores[0], o_scores)


def test_continuous_bench_clip_has_no_cuts(nets):
    import bench
    bench.select_workload('bd4')
    n, (c, h, w) = bench.CLIPS_PER_GPU, bench.LR
    clips = bench.synthetic_clips(n, 24, seed=100).numpy()
    u8 = np.ascontiguousarray(np.rint(clips * 255.0).astype(np.uint8).transpose(0, 1, 3, 4, 2))
    net = nets['bd4']
    want, _, _ = _push(net.stream(n, h, w, device=DEV), u8, [16, 8], 'host')
    got, cuts, scores = _push(net.stream(n, h, w, device=DEV, scene_cut=THR), u8, [16, 8], 'host')
    assert np.array_equal(got, want)
    assert not cuts.any(), scores.max()
    for k in range(n):
        assert np.array_equal(scores[k], S.stream(u8[k].astype(np.float32) / np.float32(255), set(), THR)[0])


def test_scene_cut_adds_two_launches_per_step(nets):
    net, h, w = nets['bd4'], BD4['h'], BD4['w']
    rgb = _two_shot_rgb(h, w)[:, :1]
    for kw in (dict(), dict(input='nv12', out_format='p010'), dict(out_size=(402, 960))):
        frames = C.rgb_to_yuv(rgb, 'nv12', 'bt601') if kw.get('input') == 'nv12' else rgb
        plain = net.stream(2, h, w, device=DEV, **kw)
        plain.push(frames)
        det = net.stream(2, h, w, device=DEV, scene_cut=THR, **kw)
        det.push(frames)
        assert det._engine.launches_per_step == plain._engine.launches_per_step + 2, kw
        plain.close()
        det.close()
