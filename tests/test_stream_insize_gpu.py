"""pytest -m gpu: streams at any input resolution -- tg_stream_frame_in_resample (decode + resize + slot reset in one
launch) against the float64 oracle and, bit for bit, against the frame input at source size followed by
tg_resample_nchw_f32; and FRNet.stream(in_size=) against an input='float32' stream pushed those resized frames.

The net's LR frame is oracle/resample.resize(decode(picture), (hn, wn), filter) in fp32, decode being the frame
input's (uint8 / 255, or the YUV conversion of oracle/yuv_color.py / oracle/yuv_422_444.py; 10 bit / 1023)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import frame_window as FW          # noqa: E402
from oracle import resample as R               # noqa: E402
from oracle import yuv_422_444 as Y            # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
F32_TOL = 4e-6                  # tests/test_resample_gpu.py's bound for the fp32 resize against float64
GUARD = 64                      # guard words around the source frames and the output
THR = 10.0

# (layout, channel order / colour): uint8 RGB and BGR, every YUV layout, BT.601 and BT.709, limited and full range
SOURCES = [('rgb', 'bt601'), ('bgr', 'bt601'), ('nv12', 'bt601'), ('nv12', 'bt709-full'), ('i420', 'bt709'),
           ('i420', 'bt601-full'), ('p010', 'bt709'), ('p010', 'bt601-full'), ('i420_10', 'bt601'),
           ('i420_10', 'bt709-full'), ('yuy2', 'bt601'), ('yuy2', 'bt709-full'), ('uyvy', 'bt709'),
           ('uyvy', 'bt601-full'), ('i444', 'bt601-full'), ('i444', 'bt709'), ('i444_10', 'bt709'),
           ('i444_10', 'bt601-full')]
H, W = 36, 52                   # the source picture: ragged (52 is no tile multiple), anamorphic ratios below
# per axis 1/4, 1/2, 3/4, 1, 4/3 and 2, paired with a different ratio on the other axis
SIZES = [(9, 26), (18, 39), (27, 52), (36, 69), (48, 104), (72, 13)]
CROP = (4, 6)                   # the picture's place in frames of (H + 10) x (W + 14)


@pytest.fixture(scope='module')
def net():
    n = T.FRNet(3, 3, 64, 2, 'BD', 4)
    n.load_state_dict(synthetic.make_frnet_params(0, nb=2, gain=1.0), strict=True)
    return n.to(DEV).eval()


def _layout(src):
    return 'rgb' if src in ('rgb', 'bgr') else src


def _encode(rgb, layout, color):
    """RGB uint8 [..., h, w, 3] -> frames of the layout (10 bit from the fp32 codes / 255)."""
    if layout == 'rgb':
        return rgb
    if Y.depth_of(layout) == 8:
        return Y.rgb_to_yuv(rgb, layout, color)
    return Y.rgb_f32_to_yuv(rgb.astype(np.float32) / 255, layout, color)


def _random_frames(src, color, n, fh, fw, seed):
    """n stored frames of every word value the layout has (10 bit: 0..1023, P010 << 6)."""
    rng = np.random.default_rng(seed)
    layout = _layout(src)
    if layout == 'rgb':
        return rng.integers(0, 256, (n, fh, fw, 3), dtype=np.uint8)
    top = 1024 if Y.depth_of(layout) == 10 else 256
    v = rng.integers(0, top, (n, *Y.frame_shape(layout, fh, fw))).astype(Y.word_dtype(layout))
    return (v << 6).astype(np.uint16) if layout == 'p010' else v


def _decode(frames, src, color, box):
    """float64 [n,3,h,w]: the picture `box` of each frame as the frame input decodes it (oracle)."""
    layout = _layout(src)
    out = []
    for f in frames:
        pic = FW.crop_words(f, layout, *box)
        if layout == 'rgb':
            rgb = pic[..., ::-1] if src == 'bgr' else pic
            scale = 255.0
        else:
            rgb = Y.yuv_to_rgb(pic, layout, color)
            scale = 1023.0 if Y.depth_of(layout) == 10 else 255.0
        out.append(rgb.astype(np.float64).transpose(2, 0, 1) / scale)
    return np.stack(out)


def _guarded(frames):
    """frames on the device inside a buffer whose GUARD words before and after are all-ones (the largest sample)."""
    t = torch.from_numpy(np.ascontiguousarray(frames))
    flat = t.reshape(-1)
    wide = flat.view(torch.int16) if flat.dtype == torch.uint16 else flat
    buf = torch.full((flat.numel() + 2 * GUARD,), -1 if wide.dtype == torch.int16 else 255, dtype=wide.dtype,
                     device=DEV)
    buf[GUARD:GUARD + flat.numel()].copy_(wide)
    region = buf[GUARD:GUARD + flat.numel()]
    return (region.view(torch.uint16) if flat.dtype == torch.uint16 else region).view(t.shape)


def _tables(h, w, hn, wn, filt):
    return [tuple(t.to(DEV) for t in ops.resample_table(a, b, filt)) for a, b in ((h, hn), (w, wn))]


def _fused(frames_dev, src, color, box, size, filt, reset=None, lr_prev=None, hr_prev=None):
    """tg_stream_frame_in_resample into a NaN buffer: (lr fp32 [n,3,hn,wn] on the host, guard bands untouched)."""
    n = frames_dev.shape[0]
    hn, wn = size
    layout = _layout(src)
    count = n * 3 * hn * wn
    buf = torch.full((count + 2 * GUARD,), float('nan'), device=DEV)
    before = buf.view(torch.int32).clone()
    lr = buf[GUARD:GUARD + count].view(n, 3, hn, wn)
    lp = torch.zeros(n, 3, hn, wn, device=DEV) if lr_prev is None else lr_prev
    hp = torch.zeros(n, 3, 4 * hn, 4 * wn, device=DEV) if hr_prev is None else hr_prev
    ops.stream_frame_in_resample(frames_dev, None if layout == 'rgb' else layout, color, reset, lr, lp, hp, 4,
                                 *_tables(box[2], box[3], hn, wn, filt), box[2:], bgr=src == 'bgr', window=box[:2])
    torch.cuda.synchronize()
    bits = buf.view(torch.int32)
    guard = torch.equal(bits[:GUARD], before[:GUARD]) and torch.equal(bits[GUARD + count:], before[GUARD + count:])
    return lr.cpu().numpy(), guard


def _two_launches(frames_dev, src, color, box, size, filt):
    """The existing frame input at source size into a scratch frame, then tg_resample_nchw_f32 with fp32 output."""
    n = frames_dev.shape[0]
    h, w = box[2:]
    layout = _layout(src)
    scratch = torch.empty(n, 3, h, w, device=DEV)
    lp, hp = torch.zeros(n, 3, h, w, device=DEV), torch.zeros(n, 3, 4 * h, 4 * w, device=DEV)
    if layout == 'rgb':
        ops.stream_frame_in(frames_dev, None, scratch, lp, hp, 4, src == 'bgr', window=box[:2])
    else:
        ops.stream_frame_in_yuv(frames_dev, layout, color, None, scratch, lp, hp, 4, window=box[:2])
    out = torch.empty(n, 3, *size, device=DEV)
    ops.resample(scratch, *_tables(h, w, *size, filt), out_f32=out)
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize('filt', R.FILTERS)
@pytest.mark.parametrize('src, color', SOURCES)
def test_kernel_matches_oracle_and_the_two_launches(src, color, filt):
    for cropped in (False, True):
        fh, fw = (H + 10, W + 14) if cropped else (H, W)
        box = (*CROP, H, W) if cropped else (0, 0, H, W)
        frames = _random_frames(src, color, 2, fh, fw, seed=fh * 7 + len(src) + len(color))
        dev = _guarded(frames)
        pic = _decode(frames, src, color, box)
        for size in SIZES:
            got, guard = _fused(dev, src, color, box, size, filt)
            assert guard, (cropped, size)
            err = np.abs(got.astype(np.float64) - R.resize(pic, size, filt))
            assert err.max() <= F32_TOL, (cropped, size, float(err.max()))    # NaN (an outside read) fails too
            again, _ = _fused(dev, src, color, box, size, filt)
            assert np.array_equal(got.view(np.uint32), again.view(np.uint32))
            two = _two_launches(dev, src, color, box, size, filt)
            assert np.array_equal(got.view(np.uint32), two.view(np.uint32)), (cropped, size)


@pytest.mark.parametrize('src, color', [('rgb', 'bt601'), ('nv12', 'bt709'), ('i444_10', 'bt601-full')])
def test_reset_zeroes_the_flagged_slots_only(src, color):
    n, size = 3, (54, 78)
    frames = _random_frames(src, color, n, 72, 104, seed=5)
    rng = np.random.default_rng(6)
    lp0 = torch.from_numpy(rng.standard_normal((n, 3, *size), dtype=np.float32)).to(DEV)
    hp0 = torch.from_numpy(rng.standard_normal((n, 3, 4 * size[0], 4 * size[1]), dtype=np.float32)).to(DEV)
    box = (0, 0, 72, 104)
    for mask in ([1, 0, 1], [0, 0, 0], [0, 1, 0]):
        lp, hp = lp0.clone(), hp0.clone()
        reset = torch.tensor(mask, dtype=torch.int32, device=DEV)
        got, guard = _fused(_guarded(frames), src, color, box, size, 'bicubic', reset, lp, hp)
        assert guard
        plain, _ = _fused(_guarded(frames), src, color, box, size, 'bicubic')
        assert np.array_equal(got.view(np.uint32), plain.view(np.uint32))      # the reset does not touch lr_curr
        for k, m in enumerate(mask):
            if m:
                assert not lp[k].any() and not hp[k].any() and not torch.signbit(hp[k]).any()
            else:
                assert torch.equal(lp[k].view(torch.int32), lp0[k].view(torch.int32))
                assert torch.equal(hp[k].view(torch.int32), hp0[k].view(torch.int32))


# ------------------------------------------------------------------------------------------------- streams
def _clip(src, color, n, k, fh, fw, seed, cut_at=None):
    """[n,k,*frame] stored frames: a smooth picture moving one pixel a frame, a hard cut (inverted picture) at
    frame cut_at."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        base = rng.integers(0, 256, (fh // 2 + 1, fw // 2 + 1, 3))
        clip = []
        for i in range(k):
            b = base if cut_at is None or i < cut_at else 255 - base
            rgb = np.roll(np.repeat(np.repeat(b, 2, 0), 2, 1)[:fh, :fw], i, axis=1).astype(np.uint8)
            clip.append(_encode(rgb[..., ::-1] if src == 'bgr' else rgb, _layout(src), color))
        out.append(np.stack(clip))
    return np.ascontiguousarray(np.stack(out))


def _lr_frames(frames, src, color, box, size, filt):
    """The fp32 LR frames [n,k,3,hn,wn] of (2): what an input='float32' stream is pushed."""
    n, k = frames.shape[:2]
    out = [_fused(_guarded(frames[:, i]), src, color, box, size, filt)[0] for i in range(k)]
    return np.ascontiguousarray(np.stack(out, 1))


def _chunks(frames):
    """3 frames, a 1-frame push that resets slot 0, the rest."""
    n = frames.shape[0]
    return [(frames[:, :3], None), (frames[:, 3:4], [True] + [False] * (n - 1)), (frames[:, 4:], None)]


def _run(stream, chunks, out='host', flush=False):
    res, cuts, scores = [], [], []
    pushes = [lambda f=f, r=r: stream.push(f, reset=r, out=out) for f, r in chunks]
    if flush:
        pushes.append(lambda: stream.flush(out=out))
    for push in pushes:
        r = push()
        res.append(r.cpu().numpy() if out == 'device' else r)
        if stream.last_cuts is not None:
            c, s = stream.last_cuts, stream.last_scores
            cuts.append(c.cpu().numpy() if out == 'device' else c)
            scores.append(s.cpu().numpy() if out == 'device' else s)
    cat = lambda xs: np.concatenate(xs, 1) if xs else None       # noqa: E731
    return cat(res), cat(cuts), cat(scores)


# (source layout, colour, frame h x w, crop box or None, in_size, filter, stream keywords, out)
ARMS = {
    'rgb': ('rgb', 'bt601', (36, 52), None, (27, 39), 'lanczos', {}, 'host'),
    'nv12-out_size': ('nv12', 'bt601', (36, 52), None, (18, 26), 'bicubic',
                      dict(out_format='nv12', out_size=(60, 80)), 'device'),
    'p010': ('p010', 'bt709', (36, 52), None, (48, 70), 'bicubic', dict(out_format='p010', out_color='bt709'),
             'host'),
    'crop-out_frame': ('bgr', 'bt601', (44, 66), (4, 6, 36, 52), (27, 39), 'bicubic',
                       dict(out_frame=(120, 170)), 'host'),
    'scene_cut': ('nv12', 'bt709-full', (36, 52), None, (24, 40), 'lanczos', dict(scene_cut=THR), 'host'),
    'pad-reflect': ('i420', 'bt601', (36, 52), None, (18, 26), 'bicubic',
                    dict(pad_front=5, padding_mode='reflect', scene_cut=THR), 'host'),
    'pad-replicate': ('yuy2', 'bt601', (36, 52), None, (45, 65), 'bicubic',
                      dict(pad_front=5, padding_mode='replicate'), 'host'),
}


@pytest.mark.parametrize('arm', list(ARMS))
def test_stream_equals_float32_stream_of_the_resized_frames(net, arm):
    src, color, (fh, fw), crop, size, filt, kw, out = ARMS[arm]
    n, k = 2, 9
    box = crop or (0, 0, fh, fw)
    frames = _clip(src, color, n, k, fh, fw, seed=len(arm), cut_at=6)
    lr = _lr_frames(frames, src, color, box, size, filt)
    input = 'uint8' if _layout(src) == 'rgb' else src
    color_kw = {} if input == 'uint8' else dict(in_color=color)
    flush = 'pad_front' in kw
    got = _run(net.stream(n, fh, fw, input=input, channel_order='bgr' if src == 'bgr' else 'rgb', crop=crop,
                          in_size=size, in_filter=filt, **color_kw, **kw), _chunks(frames), out, flush)
    want = _run(net.stream(n, *size, input='float32', **kw), _chunks(lr), out, flush)
    assert got[0].shape[1] == k
    for g, w in zip(got, want):             # frames, cuts, scores
        if w is None:
            assert g is None
        else:
            np.testing.assert_array_equal(g, w)
    assert (got[1] is not None) == ('scene_cut' in kw)


@pytest.mark.parametrize('input', ['uint8', 'nv12', 'p010'])
def test_launch_count_and_the_identity_size(net, input):
    n, fh, fw, size = 2, 36, 52, (18, 26)
    src = 'rgb' if input == 'uint8' else input
    frames = _clip(src, 'bt601', n, 4, fh, fw, seed=3)
    resized = net.stream(n, fh, fw, input=input, in_size=size)
    resized.push(frames)
    small = net.stream(n, *size, input=input)
    small.push(_clip(src, 'bt601', n, 2, *size, seed=4))
    assert resized._engine.launches_per_step == small._engine.launches_per_step
    # in_size equal to the picture: the plain stream, launch for launch and byte for byte
    same = net.stream(n, fh, fw, input=input, in_size=(fh, fw), in_filter='lanczos')
    plain = net.stream(n, fh, fw, input=input)
    a, b = same.push(frames), plain.push(frames)
    np.testing.assert_array_equal(a, b)
    assert same._engine.launches_per_step == plain._engine.launches_per_step
    assert same._engine.in_tables is None
