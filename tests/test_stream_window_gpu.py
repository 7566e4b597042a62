"""pytest -m gpu: picture windows of streamed video -- FRNet.stream(crop=, out_frame=, out_origin=), the windowed
kernels behind them (tg_stream_frame_in[_yuv]_window, tg_rgb_to_yuv_window, tg_float_to_uint8_nhwc_window,
tg_resample_nchw_f32_window), tg_fill_black and tg_luma_line_sums / detect_bars.

oracle/frame_window.py is the specification: a cropped stream equals the plain stream over the host-cropped frames,
a padded output equals the plain output placed into the format's black, byte for byte."""
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
from oracle import yuv_422_444 as Y            # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
GUARD = 0xAB
THR = 10.0


@pytest.fixture(scope='module')
def net():
    n = T.FRNet(3, 3, 64, 2, 'BD', 4)
    n.load_state_dict(synthetic.make_frnet_params(0, nb=2, gain=1.0), strict=True)
    return n.to(DEV).eval()


def _layout(input):
    return 'rgb' if input == 'uint8' else input


def _clip(input, n, k, Hf, Wf, box, seed, cut_at=None):
    """Stored frames [n,k,*frame] of the input layout: seeded noise everywhere (bars included) and a smoother moving
    picture in the box, with a hard cut at frame cut_at."""
    rng = np.random.default_rng(seed)
    layout = _layout(input)
    out = np.empty((n, k, *FW.frame_shape(layout, Hf, Wf)), Y.word_dtype(layout) if layout != 'rgb' else np.uint8)
    top, left, ch, cw = box
    for j in range(n):
        base = rng.integers(0, 256, (ch // 2 + 1, cw // 2 + 1, 3))
        for i in range(k):
            b = base if cut_at is None or i < cut_at else 255 - base
            pic = np.repeat(np.repeat(b, 2, 0), 2, 1)[:ch, :cw]
            pic = np.roll(pic, i, axis=1).astype(np.uint8)
            if layout == 'rgb':
                frame = rng.integers(0, 256, (Hf, Wf, 3), dtype=np.uint8)
                frame[top:top + ch, left:left + cw] = pic
            else:
                noise = rng.integers(0, 256, (Hf, Wf, 3), dtype=np.uint8)
                noise[top:top + ch, left:left + cw] = pic
                frame = Y.rgb_to_yuv(noise, layout) if Y.depth_of(layout) == 8 else \
                    Y.rgb_f32_to_yuv(noise.astype(np.float32) / 255, layout)
            out[j, i] = frame
    return out


def _crop(frames, input, box):
    layout = _layout(input)
    n, k = frames.shape[:2]
    return np.stack([np.stack([FW.crop_words(frames[j, i], layout, *box) for i in range(k)]) for j in range(n)])


def _run(stream, chunks, out='host'):
    """push every (frames, reset) chunk; the outputs concatenated along k, and the scene-cut reports."""
    res, cuts, scores = [], [], []
    for frames, reset in chunks:
        r = stream.push(frames, reset=reset, out=out)
        res.append(r.cpu().numpy() if out == 'device' else r)
        if stream.last_cuts is not None:
            c, s = stream.last_cuts, stream.last_scores
            cuts.append(c.cpu().numpy() if out == 'device' else c)
            scores.append(s.cpu().numpy() if out == 'device' else s)
    cat = lambda xs: np.concatenate(xs, 1) if xs else None       # noqa: E731
    return cat(res), cat(cuts), cat(scores)


def _chunks(frames):
    """3 frames, a 1-frame push that resets slot 0, the rest."""
    n = frames.shape[0]
    return [(frames[:, :3], None), (frames[:, 3:4], [True] + [False] * (n - 1)), (frames[:, 4:], None)]


CROP_INPUTS = [('uint8', 'rgb', 'bt601'), ('uint8', 'bgr', 'bt601'), ('nv12', 'rgb', 'bt601'),
               ('i420', 'rgb', 'bt709'), ('p010', 'rgb', 'bt709-full'), ('i420_10', 'rgb', 'bt601'),
               ('yuy2', 'rgb', 'bt601'), ('uyvy', 'rgb', 'bt601-full'), ('i444', 'rgb', 'bt709'),
               ('i444_10', 'rgb', 'bt601')]


@pytest.mark.parametrize('input, order, color', CROP_INPUTS)
@pytest.mark.parametrize('out', ['host', 'device'])
def test_crop_equals_plain_stream_over_cropped_frames(net, input, order, color, out):
    Hf, Wf = 28, 40
    gy, gx = FW.grid(_layout(input))
    box = (4, 6, 16, 24) if gy == 2 or gx == 2 else (5, 7, 17, 23)
    frames = _clip(input, 2, 7, Hf, Wf, box, 11, cut_at=5)
    kw = dict(input=input, channel_order=order, in_color=color, scene_cut=THR)
    got = _run(net.stream(2, Hf, Wf, crop=box, **kw), _chunks(frames), out)
    want = _run(net.stream(2, box[2], box[3], **kw), _chunks(_crop(frames, input, box)), out)
    for g, w in zip(got, want):             # frames, cuts, scores
        np.testing.assert_array_equal(g, w)


@pytest.mark.parametrize('layout', ['nv12', 'p010'])
def test_pitched_decoder_surface(net, layout):
    """A mapped NVDEC surface: pitch 512 words, 144 rows, the 134 x 320 picture at its top-left, chroma at
    pitch * 144, everything else 0xAB -- read as the (144, 512) frame with crop=(0, 0, 134, 320)."""
    h, w, pitch, rows = 134, 320, 512, 144
    packed = _clip(layout, 1, 3, h, w, (0, 0, h, w), 5)
    dt = Y.word_dtype(layout)
    surf = np.full((1, 3, rows * 3 // 2, pitch), 0xABAB if dt == np.uint16 else GUARD, dt)
    surf[:, :, :h, :w] = packed[:, :, :h]
    surf[:, :, rows:rows + h // 2, :w] = packed[:, :, h:]
    got = net.stream(1, rows, pitch, input=layout, crop=(0, 0, h, w)).push(surf)
    want = net.stream(1, h, w, input=layout).push(packed)
    np.testing.assert_array_equal(got, want)


PAD_OUTPUTS = [('rgb', 'bt601'), ('nv12', 'bt601'), ('i420', 'bt709'), ('p010', 'bt601'), ('p010', 'bt709-full'),
               ('i420_10', 'bt601-full'), ('yuy2', 'bt601'), ('uyvy', 'bt709'), ('i444', 'bt601-full'),
               ('i444_10', 'bt601')]


@pytest.mark.parametrize('out_format, color', PAD_OUTPUTS)
@pytest.mark.parametrize('out_size', [None, (48, 100)])
def test_out_frame_is_the_plain_output_placed_in_black(net, out_format, color, out_size):
    h, w = 16, 24
    Ho, Wo = out_size or (4 * h, 4 * w)
    Hf, Wf = Ho + 22, Wo + 40
    frames = _clip('uint8', 2, 9, h, w, (0, 0, h, w), 3, cut_at=6)
    chunks = _chunks(frames) + [(frames[:, :2], [False, True])]
    kw = dict(out_format=out_format, out_color=color, out_size=out_size, scene_cut=THR)
    padded = net.stream(2, h, w, out_frame=(Hf, Wf), **kw)
    got = _run(padded, chunks)
    want = _run(net.stream(2, h, w, **kw), chunks)
    y, x = padded.out_origin
    layout = _layout(out_format) if out_format != 'rgb' else 'rgb'
    n, k = want[0].shape[:2]
    placed = np.stack([np.stack([FW.place_words(want[0][j, i], layout, color, Hf, Wf, y, x) for i in range(k)])
                       for j in range(n)])
    np.testing.assert_array_equal(got[0], placed)
    np.testing.assert_array_equal(got[1], want[1])


def test_crop_and_out_frame_together_keep_the_launch_count(net):
    Hf, Wf, box = 28, 40, (6, 0, 16, 40)
    frames = _clip('nv12', 2, 3, Hf, Wf, box, 7)
    plain = net.stream(2, 16, 40, input='nv12', out_format='nv12')
    both = net.stream(2, Hf, Wf, input='nv12', out_format='nv12', crop=box, out_frame=(96, 180))
    want = plain.push(_crop(frames, 'nv12', box))
    got = both.push(frames)
    assert both._engine.launches_per_step == plain._engine.launches_per_step
    y, x = both.out_origin
    for i in range(3):
        np.testing.assert_array_equal(got[1, i], FW.place_words(want[1, i], 'nv12', 'bt601', 96, 180, y, x))
    rgb = _clip('uint8', 2, 1, Hf, Wf, box, 1)
    for kw in (dict(), dict(out_size=(32, 80))):
        a = net.stream(2, 16, 40, **kw)
        b = net.stream(2, Hf, Wf, crop=box, out_frame=(100, 200), **kw)
        a.push(_crop(rgb, 'uint8', box))
        b.push(rgb)
        assert a._engine.launches_per_step == b._engine.launches_per_step


# ------------------------------------------------------------------------------------------------- kernels
def _guarded(shape, dtype, offset=3):
    """A tensor of `shape` inside a 0xAB byte buffer, `offset` words in (so most windows are not 16-byte aligned;
    packed 4:2:2 frames keep their 4-byte alignment with offset 4)."""
    size = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
    esz = torch.tensor([], dtype=dtype).element_size()
    buf = torch.full((offset * esz + size + 64,), GUARD, dtype=torch.uint8, device=DEV)
    return buf, buf[offset * esz:offset * esz + size].view(dtype).view(shape)


# frames of 14 x 32, pictures of 8 x 20: top-left, inside, bottom-right corner, odd (RGB and 4:4:4 only)
WINDOWS = [(0, 0), (2, 4), (6, 12), (1, 3)]


@pytest.mark.parametrize('layout', FW.LAYOUTS)
def test_windowed_frame_in_kernel(layout):
    Hf, Wf, h, w = 14, 32, 8, 20
    gy, gx = FW.grid(layout)
    rng = np.random.default_rng(1)
    dt = np.uint8 if layout == 'rgb' else Y.word_dtype(layout)
    frames = rng.integers(0, 1 << 16 if dt == np.uint16 else 256, (2, *FW.frame_shape(layout, Hf, Wf)), dtype=dt)
    tdt = torch.uint16 if dt == np.uint16 else torch.uint8
    _, src = _guarded(frames.shape, tdt, 4 if layout in Y.LAYOUTS_422 else 3)
    src.copy_(torch.from_numpy(frames))
    lr = torch.full((2, 3, h, w), float('nan'), device=DEV)
    lp, hp = torch.zeros_like(lr), torch.zeros(2, 3, 4 * h, 4 * w, device=DEV)
    for top, left in WINDOWS:
        if top % gy or left % gx:
            continue
        crop = np.stack([FW.crop_words(f, layout, top, left, h, w) for f in frames])
        want = torch.full_like(lr, float('nan'))
        if layout == 'rgb':
            ops.stream_frame_in(src, None, lr, lp, hp, 4, window=(top, left))
            ops.stream_frame_in(torch.from_numpy(crop).to(DEV), None, want, lp, hp, 4)
        else:
            ops.stream_frame_in_yuv(src, layout, 'bt709', None, lr, lp, hp, 4, window=(top, left))
            ops.stream_frame_in_yuv(torch.from_numpy(crop).to(DEV), layout, 'bt709', None, want, lp, hp, 4)
        torch.testing.assert_close(lr, want, rtol=0, atol=0)


@pytest.mark.parametrize('layout', FW.LAYOUTS)
def test_windowed_writers_touch_only_the_picture(layout):
    H, W, Hf, Wf = 8, 20, 14, 32
    gy, gx = FW.grid(layout)
    rng = np.random.default_rng(2)
    f32 = torch.from_numpy(rng.uniform(-0.05, 1.05, (2, 3, H, W)).astype(np.float32)).to(DEV)
    u8 = ops.float_to_uint8_nhwc(f32)
    ten = layout != 'rgb' and Y.depth_of(layout) == 10
    dt = torch.uint16 if ten else torch.uint8
    fshape = FW.frame_shape(layout, Hf, Wf)
    # RGB: 3 bytes in, the per-pixel uint8 writer; 4 bytes in (4-byte aligned, with frame width and every even window's
    # left edge multiples of 4), the 4-pixel c3x4 writer
    offsets = (3, 4) if layout == 'rgb' else (4,) if layout in Y.LAYOUTS_422 else (3,)
    for (top, left), off in [(wd, o) for wd in WINDOWS for o in offsets]:
        if top % gy or left % gx:
            continue
        buf, out = _guarded((2, *fshape), dt, off)
        before = buf.clone()
        if layout == 'rgb':
            ops.float_to_uint8_nhwc_window(f32, out, (top, left))
            plain = u8
        else:
            src = dict(rgb_f32=f32) if ten else dict(rgb_u8=u8)
            ops.rgb_to_yuv(layout, 'bt601-full', out=out, window=(top, left), **src)
            plain = ops.rgb_to_yuv(layout, 'bt601-full', **src)
        got = out.cpu().numpy()
        for j in range(2):
            np.testing.assert_array_equal(FW.crop_words(got[j], layout, top, left, H, W), plain[j].cpu().numpy())
        # everything else keeps its guard bytes: place the picture into the guard frame and compare whole buffers
        mark = buf.clone()
        mark_out = mark[out.data_ptr() - buf.data_ptr():][:out.numel() * out.element_size()].view(dt).view(out.shape)
        g = before[out.data_ptr() - buf.data_ptr():][:out.numel() * out.element_size()].view(dt).view(out.shape)
        gnp = g.cpu().numpy().copy()
        for j in range(2):
            pic = plain[j].cpu().numpy()
            for (dst, rs, cs, wpc), (srcp, *_) in zip(FW._planes(gnp[j], layout, Hf, Wf),
                                                      FW._planes(pic, layout, H, W)):
                r, q = FW._slices(rs, cs, wpc, top, left, H, W)
                dst[r, q] = srcp
        mark_out.copy_(torch.from_numpy(gnp))
        assert torch.equal(buf, mark)


def test_windowed_resample_writes_only_the_picture():
    H, W, Ho, Wo, Hf, Wf = 20, 36, 31, 50, 40, 70
    x = torch.rand(2, 3, H, W, device=DEV)
    tabs = [tuple(t.to(DEV) for t in ops.resample_table(a, b, 'lanczos')) for a, b in ((H, Ho), (W, Wo))]
    plain = ops.resample(x, *tabs).cpu().numpy()
    for top, left in ((0, 0), (Hf - Ho, Wf - Wo), (3, 7)):
        buf, out = _guarded((2, Hf, Wf, 3), torch.uint8, offset=5)
        ops.resample(x, *tabs, out_u8=out, window=(top, left))
        want = np.full((2, Hf, Wf, 3), GUARD, np.uint8)
        want[:, top:top + Ho, left:left + Wo] = plain
        np.testing.assert_array_equal(out.cpu().numpy(), want)
        assert (buf[:5] == GUARD).all() and (buf[5 + out.numel():] == GUARD).all()


@pytest.mark.parametrize('layout', FW.LAYOUTS)
@pytest.mark.parametrize('color', ['bt601', 'bt709-full'])
def test_fill_black(layout, color):
    if layout == 'rgb' and color != 'bt601':
        pytest.skip('RGB black has no colour')
    Hf, Wf = 10, 14
    dt = torch.uint16 if layout != 'rgb' and Y.depth_of(layout) == 10 else torch.uint8
    off = 4 if layout in Y.LAYOUTS_422 else 3
    buf, out = _guarded((3, *FW.frame_shape(layout, Hf, Wf)), dt, off)
    ops.fill_black(out, None if layout == 'rgb' else layout, color)
    want = np.stack([FW.black_frame(layout, color, Hf, Wf)] * 3)
    np.testing.assert_array_equal(out.cpu().numpy(), want)
    assert (buf[:off * out.element_size()] == GUARD).all()
    assert (buf[off * out.element_size() + out.numel() * out.element_size():] == GUARD).all()


@pytest.mark.parametrize('layout, order', [('rgb', 'rgb'), ('rgb', 'bgr'), ('nv12', 'rgb'), ('p010', 'rgb'),
                                           ('i420_10', 'rgb'), ('yuy2', 'rgb'), ('uyvy', 'rgb'), ('i444', 'rgb'),
                                           ('i444_10', 'rgb')])
def test_luma_line_sums_and_detect_bars(layout, order):
    input = 'uint8' if layout == 'rgb' else layout
    Hf, Wf, box = 60, 300, (8, 20, 44, 260)
    frames = _clip(input, 1, 4, Hf, Wf, box, 9)[0]
    # the bars of _clip hold full-range noise: darken them (RGB <= 5: luma <= 20 even at limited range) and
    # brighten the picture (RGB >= 60)
    rgb = frames if layout == 'rgb' else Y.yuv_to_rgb(frames, layout)
    if layout != 'rgb' and Y.depth_of(layout) == 10:
        rgb = rgb >> 2
    mask = np.zeros((Hf, Wf), bool)
    mask[box[0]:box[0] + box[2], box[1]:box[1] + box[3]] = True
    rgb = np.where(mask[..., None], np.maximum(rgb, 60), rgb % 6).astype(np.uint8)
    if layout == 'rgb':
        frames = rgb
    elif Y.depth_of(layout) == 8:
        frames = Y.rgb_to_yuv(rgb, layout)
    else:
        frames = Y.rgb_f32_to_yuv(rgb.astype(np.float32) / 255, layout)
    dev = torch.from_numpy(np.ascontiguousarray(frames)).to(DEV)
    rows, cols = ops.luma_line_sums(dev, None if layout == 'rgb' else layout, order == 'bgr')
    wr, wc = FW.line_sums(frames, layout, order)
    np.testing.assert_array_equal(rows.cpu().numpy(), wr)
    np.testing.assert_array_equal(cols.cpu().numpy(), wc)
    got = T.detect_bars(dev, input=input, channel_order=order)
    assert got == FW.detect_bars(frames, layout, order)
    assert got == box
    assert T.detect_bars(torch.zeros_like(dev), input=input) == (0, 0, Hf, Wf)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two devices')
def test_padded_stream_and_detect_bars_on_a_device_that_is_not_current(net):
    """The black fill of out_frame and detect_bars run on the stream's / the frames' device, not the current one."""
    h, w = 16, 24
    frames = _clip('uint8', 1, 3, h, w, (0, 0, h, w), 4)
    kw = dict(out_format='nv12', out_frame=(80, 120))
    want = net.stream(1, h, w, **kw).push(frames)
    dev1 = torch.device('cuda', 1)
    net1 = T.FRNet(3, 3, 64, 2, 'BD', 4)
    net1.load_state_dict(net.state_dict(), strict=True)
    net1 = net1.to(dev1).eval()
    box = (6, 0, 28, 64)
    letterboxed = np.zeros((2, 40, 64, 3), np.uint8)
    letterboxed[:, 6:34] = 200
    with torch.cuda.device(0):
        got = net1.stream(1, h, w, device=dev1, **kw).push(frames)
        bars = T.detect_bars(torch.from_numpy(letterboxed).to(dev1))
    np.testing.assert_array_equal(got, want)
    assert bars == box
