"""pytest -m gpu: 10-bit 4:2:2 (P210, I422_10, v210) frame I/O of streamed inference -- tg_stream_frame_in_yuv,
tg_rgb_to_yuv, their window variants, tg_stream_frame_in_resample, tg_fill_black and tg_luma_line_sums for the new
layouts, and FRNet.stream(input=, out_format=) with them, alone and with in_size=, out_size=, crop=, out_frame=,
scene_cut= and pad_front=.

The specification is oracle/yuv_422_10.py; every kernel output below equals it bit for bit.  Heights are odd and
widths no multiple of 6 or 48, so v210 rows end in partial groups and padding.  Output buffers are filled with NaN
or sit inside a 0xAB guard band first.  Stream inputs are anchored on the existing I444_10 path: a 4:2:2 frame
decodes as the I444_10 frame of the same samples with each pair's chroma repeated."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import yuv_422_10 as V             # noqa: E402
from oracle import yuv_422_444 as Q            # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
engine = sys.modules['tecogan-pytorch_b200.engine']
DEV = torch.device('cuda', 0)
GUARD = 0xAB
THR = 10.0


def _net(scale, degradation):
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def bi2_net():
    return _net(2, 'BI')


@pytest.fixture(scope='module')
def bd4_net():
    return _net(4, 'BD')


def _guarded(frames, offset=16):
    """frames (numpy) copied into a device buffer of 0xAB with `offset` bytes before and 64 after; (buf, view)."""
    raw = np.ascontiguousarray(frames).view(np.uint8).reshape(-1)
    buf = torch.full((offset + raw.size + 64,), GUARD, dtype=torch.uint8, device=DEV)
    region = buf[offset:offset + raw.size]
    region.copy_(torch.from_numpy(raw))
    t = region if frames.dtype == np.uint8 else region.view(torch.uint16)
    return buf, t.view(frames.shape)


def _bits(got, want):
    assert got.dtype == np.float32 and got.shape == want.shape
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist())


def _f32(rgb10):
    """RGB10 codes [..., h, w, 3] -> the stream's fp32 input [..., 3, h, w]."""
    x = rgb10.astype(np.float32) / np.float32(1023.0)
    return np.ascontiguousarray(np.moveaxis(x, -1, -3))


def _decode(frames_dev, layout, color, n, h, w, window=None):
    lr = torch.full((n, 3, h, w), float('nan'), device=DEV)
    prev = torch.full_like(lr, 3.0)
    hr = torch.full((n, 3, 2 * h, 2 * w), 5.0, device=DEV)
    ops.stream_frame_in_yuv(frames_dev, layout, color, None, lr, prev, hr, 2, window=window)
    torch.cuda.synchronize()
    return lr.cpu().numpy()


def _random(rng, n, h, w):
    return rng.integers(0, 1024, (n, h, w)), rng.integers(0, 1024, (n, h, w // 2)), rng.integers(0, 1024, (n, h, w // 2))


def _as_i444_10(y, u, v):
    """The I444_10 frames of the same samples, each pair's chroma repeated."""
    return Q.join_planes(y, np.repeat(u, 2, axis=-1), np.repeat(v, 2, axis=-1), 'i444_10')


# ------------------------------------------------------------------------------------------------ decode kernels
@pytest.mark.parametrize('color', V.COLORS)
@pytest.mark.parametrize('layout', V.LAYOUTS)
def test_kernel_decode_pattern(layout, color):
    """Every (U, V) of samples10()^2 with Y cycling through samples10(), junk in v210's bits 30-31 and row padding,
    P210's low 6 bits and I422_10 words above 1023; odd h, w = 80."""
    frames, h, w, _ = V.yuv10_pattern(layout)
    _, dev = _guarded(frames)
    got = _decode(dev, layout, color, frames.shape[0], h, w)
    _bits(got, _f32(V.yuv_to_rgb(frames, layout, color, w)))


@pytest.mark.parametrize('n,h,w', [(3, 37, 54), (2, 5, 602), (1, 1, 2), (2, 3, 1030), (1, 7, 96)])
def test_three_layouts_decode_alike_and_as_the_oracle(n, h, w):
    rng = np.random.default_rng(h * w)
    y, u, v = _random(rng, n, h, w)
    ref = None
    for color in ('bt709', 'bt601-full'):
        for layout in V.LAYOUTS:
            frames = V.join_planes(y, u, v, layout)
            _, dev = _guarded(frames, 16 if layout == 'v210' else 6)
            got = _decode(dev, layout, color, n, h, w)
            _bits(got, _f32(V.yuv_to_rgb(frames, layout, color, w)))
            if layout == 'p210':
                ref = got
            _bits(got, ref)
        _, dev = _guarded(_as_i444_10(y, u, v))
        _bits(_decode(dev, 'i444_10', color, n, h, w), ref)


@pytest.mark.parametrize('layout', V.LAYOUTS)
def test_kernel_decode_windows(layout):
    rng = np.random.default_rng(2)
    n, fh, fw = 2, 9, 50
    frames = V.join_planes(*_random(rng, n, fh, fw), layout)
    _, dev = _guarded(frames)
    for top, left, h, w in ((1, 6, 7, 18), (0, 12, 9, 38), (2, 0, 5, 50), (3, 42, 1, 8)):
        got = _decode(dev, layout, 'bt709', n, h, w, window=(top, left, fw) if layout == 'v210' else (top, left))
        want = V.decode_window(frames, layout, 'bt709', top, left, h, w, fw)
        _bits(got, _f32(want))


@pytest.mark.parametrize('layout', V.LAYOUTS)
def test_resizing_frame_input(layout):
    """tg_stream_frame_in_resample: the new layouts' per-pixel fetch gives the I444_10 result of the same samples,
    whole frame and through a window."""
    rng = np.random.default_rng(4)
    n, fh, fw = 2, 21, 62
    y, u, v = _random(rng, n, fh, fw)
    frames = V.join_planes(y, u, v, layout)
    ref444 = _as_i444_10(y, u, v)
    for window, size, out in ((None, (fh, fw), (30, 80)), ((2, 6, ), (17, 48), (13, 40)), ((0, 12), (21, 50), (9, 14))):
        res = []
        for lay, fr in ((layout, frames), ('i444_10', ref444)):
            _, dev = _guarded(fr)
            rows, cols = (tuple(t.to(DEV) for t in ops.resample_table(a, b, 'lanczos')) for a, b in zip(size, out))
            lr = torch.full((n, 3, *out), float('nan'), device=DEV)
            prev, hr = torch.zeros_like(lr), torch.zeros(n, 3, 2 * out[0], 2 * out[1], device=DEV)
            win = (*window, fw) if window and lay == 'v210' else window
            ops.stream_frame_in_resample(dev, lay, 'bt601', None, lr, prev, hr, 2, rows, cols, size, window=win)
            res.append(lr.cpu().numpy())
        _bits(res[0], res[1])


# ------------------------------------------------------------------------------------------------ encode kernels
def _hr(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(n, 3, H, W, generator=g) * 1.2 - 0.1                            # some values outside [0, 1]
    edge = torch.tensor([0.0, 1.0, 0.5 / 1023, 1.5 / 1023])                     # 0, 1 and rint's ties
    x[0, :, 0, :min(W, 4)] = edge[:min(W, 4)]
    return x


@pytest.mark.parametrize('color', V.COLORS)
@pytest.mark.parametrize('n,H,W', [(2, 37, 54), (1, 3, 530), (1, 1, 2), (2, 5, 96)])
def test_kernel_encode_whole_frames(color, n, H, W):
    """tg_rgb_to_yuv from the fp32 HR frame: the oracle's bytes inside a guard band -- v210 rows written in full,
    partial groups and padding 0 -- and the three layouts carry the same samples."""
    x = _hr(n, H, W, H * W)
    want_samples = V.encode_samples(V.quantize10(x.permute(0, 2, 3, 1).numpy()), color)
    for layout in V.LAYOUTS:
        shape = (n, *V.frame_shape(layout, H, W))
        junk = np.full(shape, GUARD, V.word_dtype(layout)) if layout == 'v210' else np.full(shape, 0xABAB, np.uint16)
        buf, out = _guarded(junk)
        ops.rgb_to_yuv(layout, color, rgb_f32=x.to(DEV), out=out)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
        want = V.rgb_f32_to_yuv(x.permute(0, 2, 3, 1).numpy(), layout, color)
        assert np.array_equal(got, want), (layout, int((got != want).sum()))
        b = buf.cpu().numpy()
        assert (b[:16] == GUARD).all() and (b[-64:] == GUARD).all(), layout
        for a, s in zip(V.split_planes(got, layout, W), want_samples):
            assert np.array_equal(a, s), layout


@pytest.mark.parametrize('layout', V.LAYOUTS)
def test_kernel_encode_windows(layout):
    """tg_rgb_to_yuv_window writes the picture's samples (v210: its groups) and no other byte."""
    n, fh, fw = 2, 11, 62
    base = np.full((n, *V.frame_shape(layout, fh, fw)), GUARD if layout == 'v210' else 0xABAB,
                   V.word_dtype(layout))
    for top, left, H, W in ((1, 6, 7, 18), (0, 0, 11, 62), (3, 42, 5, 20), (2, 12, 3, 14)):
        if layout == 'v210' and (left + W) % 6 and left + W != fw:
            continue
        x = _hr(n, H, W, 7 + left)
        buf, out = _guarded(base)
        win = (top, left, fw) if layout == 'v210' else (top, left)
        ops.rgb_to_yuv(layout, 'bt709-full', rgb_f32=x.to(DEV), out=out, window=win)
        torch.cuda.synchronize()
        want = V.encode_window(base, V.quantize10(x.permute(0, 2, 3, 1).numpy()), layout, 'bt709-full', top, left,
                               fw)
        got = out.cpu().numpy()
        assert np.array_equal(got, want), (layout, (top, left, H, W), int((got != want).sum()))
        b = buf.cpu().numpy()
        assert (b[:16] == GUARD).all() and (b[-64:] == GUARD).all()


@pytest.mark.parametrize('layout', V.LAYOUTS)
def test_fill_black_and_luma_sums(layout):
    for color in ('bt601', 'bt709-full'):
        for fh, fw in ((7, 26), (3, 96), (1, 50)):
            junk = np.full((2, *V.frame_shape(layout, fh, fw)), 0x5A, V.word_dtype(layout))
            _, out = _guarded(junk)
            if layout == 'v210':
                ops.fill_black_v210(out, color, fw)
            else:
                ops.fill_black(out, layout, color)
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy(), V.black(layout, color, fh, fw, (2,))), (color, fh, fw)
    rng = np.random.default_rng(9)
    frames = V.join_planes(*_random(rng, 3, 9, 50), layout)
    frames_dev = torch.from_numpy(frames).to(DEV)
    rows, cols = ops.luma_line_sums(frames_dev, layout, frame_w=50)
    luma = V.luma8(frames, layout, 50)
    assert np.array_equal(rows.cpu().numpy(), luma.sum(-1)) and np.array_equal(cols.cpu().numpy(), luma.sum(-2))


def test_detect_bars_v210_box_on_the_group_grid():
    h, w = 20, 62
    y = np.full((2, h, w), 64)
    y[:, 3:17, 8:59] = 700                      # picture columns [8, 59): rounds inward to [12, 54)
    f = V.join_planes(y, np.full((2, h, w // 2), 512), np.full((2, h, w // 2), 512), 'v210')
    box = engine.detect_bars(torch.from_numpy(f).to(DEV), 'v210', width=w)
    assert box == (3, 12, 14, 42)
    y[:, 3:17, 8:] = 700                        # to the right edge: the box may end inside the last group
    f = V.join_planes(y, np.full((2, h, w // 2), 512), np.full((2, h, w // 2), 512), 'v210')
    box = engine.detect_bars(torch.from_numpy(f).to(DEV), 'v210', width=w)
    assert box == (3, 12, 14, 50) and box[1] % 6 == 0
    assert engine.detect_bars(torch.from_numpy(V.join_planes(y, *[np.full((2, h, w // 2), 512)] * 2, 'p210'))
                              .to(DEV), 'p210') == (3, 8, 14, 54)


# ------------------------------------------------------------------------------------------------ streams
def _clips10(seed, n, t, h, w):
    """10-bit samples (y, u, v) [n,t,...] of synthetic clips, encoded once with the oracle."""
    clips = np.stack([synthetic.make_clip(seed + k, t, 3, h, w, shift=1 + k).numpy() for k in range(n)])
    return V.encode_samples(V.quantize10(clips.transpose(0, 1, 3, 4, 2)), 'bt709')


def _push(stream, frames, chunks, resets=None, out='host'):
    res, i = [], 0
    for j, k in enumerate(chunks):
        src = frames[:, i:i + k]
        if out == 'device':
            src = torch.from_numpy(np.ascontiguousarray(src)).to(DEV)
        o = stream.push(src, reset=resets[j] if resets else None, out=out)
        res.append(o.cpu().numpy() if isinstance(o, torch.Tensor) else o)
        i += k
    return np.concatenate(res, axis=1)


def _hr_loop(net, f32, resets):
    n, t = f32.shape[:2]
    lr = torch.from_numpy(f32).to(DEV)
    s = net.scale
    lr_prev = torch.zeros_like(lr[:, 0])
    hr_prev = torch.zeros(n, 3, s * lr.shape[3], s * lr.shape[4], device=DEV)
    outs = []
    with torch.no_grad():
        for i in range(t):
            for k in range(n):
                if (k, i) in resets:
                    lr_prev[k].zero_()
                    hr_prev[k].zero_()
            hr = net.step(lr[:, i].contiguous(), lr_prev, hr_prev)
            outs.append(hr.clone())
            lr_prev, hr_prev = lr[:, i].contiguous(), hr
    return torch.stack(outs, dim=1)


@pytest.mark.parametrize('geom', ['bd4', 'bi2'])
def test_chunked_pushes_in_and_out(geom, bd4_net, bi2_net):
    """n=2 clips of 8 frames pushed as [1,4,3] with slot 1 restarting at frame 5, host and device I/O: each layout
    in and out is the oracle's encode of the fp32 HR frames of an FRNet.step loop over the oracle's decode."""
    net = bd4_net if geom == 'bd4' else bi2_net
    h, w = (134, 320) if geom == 'bd4' else (37, 58)
    y, u, v = _clips10(31, 2, 8, h, w)
    chunks, resets, reset_at = [1, 4, 3], [None, None, [False, True]], {(1, 5)}
    colors = {'p210': 'bt709', 'i422_10': 'bt601-full', 'v210': 'bt601'}
    for layout, color in colors.items():
        frames = V.join_planes(y, u, v, layout)
        f32 = _f32(V.yuv_to_rgb(frames, layout, color, w))
        want = V.rgb_f32_to_yuv(_hr_loop(net, f32, reset_at).permute(0, 1, 3, 4, 2).cpu().numpy(), layout, color)
        for out in ('host', 'device'):
            s = net.stream(2, h, w, device=DEV, input=layout, in_color=color, out_format=layout, out_color=color)
            got = _push(s, frames, chunks, resets, out)
            s.close()
            assert got.dtype == want.dtype and np.array_equal(got, want), (layout, out, int((got != want).sum()))


@pytest.mark.parametrize('opts', ['crop', 'in_size', 'scene_cut', 'pad_front', 'crop_in_size_pad'])
def test_input_options_match_the_i444_10_stream(opts, bi2_net):
    """crop= (v210 crops on the group grid, one reaching the right edge), in_size=, scene_cut= and pad_front= on
    each new input layout: the RGB output of the I444_10 stream of the same samples, and the same cuts."""
    net = bi2_net
    h, w = 25, 62
    y, u, v = _clips10(41, 2, 7, h, w)
    y[0, 4:] = 1023 - y[0, 4:]                   # a cut in slot 0 at frame 4
    chunks, resets = [2, 1, 4], [None, [True, False], None]
    kw = {'crop': dict(crop=(2, 6, 21, 56)), 'in_size': dict(in_size=(19, 40)), 'scene_cut': dict(scene_cut=THR),
          'pad_front': dict(pad_front=2),
          'crop_in_size_pad': dict(crop=(1, 12, 23, 36), in_size=(30, 44), pad_front=3, scene_cut=THR)}[opts]
    ref444 = _as_i444_10(y, u, v)
    ref_s = net.stream(2, h, w, device=DEV, input='i444_10', in_color='bt709-full', **kw)
    ref = _push(ref_s, ref444, chunks, resets)
    ref_cuts = ref_s.last_cuts
    ref = np.concatenate([ref, ref_s.flush()], axis=1)
    for layout in V.LAYOUTS:
        s = net.stream(2, h, w, device=DEV, input=layout, in_color='bt709-full', **kw)
        got = _push(s, V.join_planes(y, u, v, layout), chunks, resets)
        cuts = s.last_cuts
        got = np.concatenate([got, s.flush()], axis=1)
        s.close()
        assert np.array_equal(got, ref), (layout, opts)
        if 'scene_cut' in kw:
            assert np.array_equal(cuts, ref_cuts), layout


def test_output_size_frame_and_origin(bi2_net):
    """out_size= and out_frame= on each new output layout: the picture carries the samples of the stream without
    out_frame (itself the encode of the resize kernel's fp32 output), the rest of the frame is black; letterbox and
    pillarbox, the v210 picture on a group edge or at the frame's right edge."""
    net = bi2_net
    h, w = 19, 30
    y, u, v = _clips10(51, 2, 4, h, w)
    frames = V.join_planes(y, u, v, 'p210')
    chunks, resets = [3, 1], [None, [False, True]]
    size = (37, 48)
    f32 = _f32(V.yuv_to_rgb(frames, 'p210', 'bt709', w))
    hr = _hr_loop(net, f32, {(1, 3)})
    tabs = [tuple(t.to(DEV) for t in ops.resample_table(a, b, 'bicubic')) for a, b in zip(hr.shape[-2:], size)]
    rs = torch.stack([ops.resample(hr[:, i].contiguous(), *tabs, out_f32=torch.empty(2, 3, *size, device=DEV))
                      for i in range(hr.shape[1])], dim=1)
    q = V.quantize10(rs.permute(0, 1, 3, 4, 2).cpu().numpy())
    for layout in V.LAYOUTS:
        s = net.stream(2, h, w, device=DEV, input='p210', in_color='bt709', out_format=layout, out_color='bt709-full',
                       out_size=size)
        plain = _push(s, frames, chunks, resets)
        s.close()
        assert np.array_equal(plain, V.rgb_to_yuv(q, layout, 'bt709-full')), layout
        # (Hf, Wf, origin): letterbox; pillarbox centred; pillarbox at the right edge (v210: 66 = 18 + 48)
        for Hf, Wf, origin in ((57, 48, None), (37, 72, None), (41, 66, (2, 18))):
            s = net.stream(2, h, w, device=DEV, input='p210', in_color='bt709', out_format=layout,
                           out_color='bt709-full', out_size=size, out_frame=(Hf, Wf), out_origin=origin)
            got = _push(s, frames, chunks, resets)
            oy, ox = s.out_origin
            s.close()
            assert ox % (6 if layout == 'v210' else 2) == 0
            want = V.black(layout, 'bt709-full', Hf, Wf, (2, 4))
            want = V.encode_window(want, q, layout, 'bt709-full', oy, ox, Wf)
            assert np.array_equal(got, want), (layout, Hf, Wf, int((got != want).sum()))


def test_single_slot_three_dim_frames(bi2_net):
    h, w = 9, 14
    y, u, v = _clips10(61, 1, 3, h, w)
    f = V.join_planes(y, u, v, 'v210')[0]                                             # [k, h, S]
    ref = bi2_net.stream(1, h, w, device=DEV, input='p210', out_format='v210').push(V.join_planes(y, u, v, 'p210'))
    got = bi2_net.stream(1, h, w, device=DEV, input='v210', out_format='v210').push(f)
    assert got.shape == (1, 3, 2 * h, 128) and np.array_equal(got, ref)
