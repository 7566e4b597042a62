"""pytest -m gpu: packed 4:2:2 (YUY2, UYVY) and planar 4:4:4 (I444, I444_10) frame I/O of streamed inference -- the
kernels tg_stream_frame_in_yuv and tg_rgb_to_yuv for the new layouts and FRNet.stream(input=, out_format=) with
them, alone and with out_size=, scene_cut= and 1-frame pushes.

The specification is oracle/yuv_422_444.py (pinned to cv2 by tests/test_stream_yuv422_444_cpu.py); every kernel
output below equals it bit for bit.  Output buffers are filled with NaN or sit inside a 0xAB guard band first."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import yuv_422_444 as C            # noqa: E402
from oracle import yuv_oracle as Y8            # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
NEW = C.LAYOUTS_422 + C.LAYOUTS_444
NEW8 = ('yuy2', 'uyvy', 'i444')
GUARD = 0xAB
THR = 10.0


def _net(scale, degradation):
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def bd4_net():
    return _net(4, 'BD')


@pytest.fixture(scope='module')
def bi2_net():
    return _net(2, 'BI')


def _placed(nbytes, offset):
    """A uint8 device buffer of 0xAB with `offset` guard bytes before and 64 after a region; returns (buf, region)."""
    buf = torch.full((offset + nbytes + 64,), GUARD, dtype=torch.uint8, device=DEV)
    return buf, buf[offset:offset + nbytes]


def _to_dev(frames, offset=0):
    raw = np.ascontiguousarray(frames).view(np.uint8).reshape(-1)
    _, region = _placed(raw.size, offset)
    region.copy_(torch.from_numpy(raw))
    t = region if frames.dtype == np.uint8 else region.view(torch.uint16)
    return t.view(frames.shape)


def _bits(got, want):
    assert got.dtype == np.float32 and got.shape == want.shape
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist())


def _decode_ref(frames, layout, color):
    rgb = C.yuv_to_rgb(frames, layout, color).astype(np.float32).transpose(0, 3, 1, 2)
    return np.ascontiguousarray(rgb / np.float32(1023.0 if C.depth_of(layout) == 10 else 255.0))


def _decode(frames_dev, layout, color, n, h, w, s=2, reset=None, prev=None, hr=None):
    lr = torch.full((n, 3, h, w), float('nan'), device=DEV)
    prev = torch.full_like(lr, 3.0) if prev is None else prev
    hr = torch.full((n, 3, s * h, s * w), 5.0, device=DEV) if hr is None else hr
    ops.stream_frame_in_yuv(frames_dev, layout, color, reset, lr, prev, hr, s)
    torch.cuda.synchronize()
    return lr, prev, hr


def _random_frames(rng, layout, n, h, w):
    dt = C.word_dtype(layout)
    return rng.integers(0, np.iinfo(dt).max + 1, size=(n, *C.frame_shape(layout, h, w))).astype(dt)


# ------------------------------------------------------------------------------------------------ decode kernel
@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('layout', NEW)
def test_kernel_decode_every_sample(layout, color):
    """8 bit: a 4096x4096 frame with every (Y, U, V) triple; I444_10: every triple of the dense sample, with 5 % of
    the words above 1023."""
    if C.depth_of(layout) == 8:
        frames = C.yuv_triples_pattern(layout)[None]
        h = w = 4096
    else:
        frames, h, w = C.yuv10_pattern(layout)
    lr, _, _ = _decode(_to_dev(frames), layout, color, frames.shape[0], h, w)
    _bits(lr.cpu().numpy(), _decode_ref(frames, layout, color))


@pytest.mark.parametrize('layout', NEW)
@pytest.mark.parametrize('n,h,w,offset', [(3, 37, 54, 4), (2, 5, 600, 12), (1, 1, 2, 0), (2, 3, 1030, 8),
                                          (1, 7, 513, 2)])
def test_kernel_decode_ragged_odd_heights(layout, n, h, w, offset):
    """Odd heights, several tiles per row (512 pixels a CTA for 4:2:2, 256 for 4:4:4), odd widths for 4:4:4, sources
    at 4-byte (4:2:2) or word offsets (odd for I444) past a 16-byte boundary; lr_prev / hr_prev untouched."""
    if layout in C.LAYOUTS_422:
        w += w % 2
        offset -= offset % 4
    elif layout == 'i444':
        offset += 1
    rng = np.random.default_rng(4000 + n * h + w + offset)
    frames = _random_frames(rng, layout, n, h, w)
    lr, prev, hr = _decode(_to_dev(frames, offset), layout, 'bt709', n, h, w, s=4)
    _bits(lr.cpu().numpy(), _decode_ref(frames, layout, 'bt709'))
    assert bool((prev == 3.0).all()) and bool((hr == 5.0).all())


@pytest.mark.parametrize('layout', NEW)
def test_kernel_decode_reset_zeroes_flagged_slots_only(layout):
    n, h, w, s = 3, 37, 54, 4
    g = torch.Generator(device=DEV).manual_seed(9)
    prev = torch.rand((n, 3, h, w), generator=g, device=DEV) + 1.0
    hr = torch.rand((n, 3, s * h, s * w), generator=g, device=DEV) + 1.0
    prev0, hr0 = prev.clone(), hr.clone()
    frames = _random_frames(np.random.default_rng(5), layout, n, h, w)
    mask = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    lr, prev, hr = _decode(_to_dev(frames), layout, 'bt601-full', n, h, w, s, reset=mask, prev=prev, hr=hr)
    for k in (0, 2):
        assert bool((prev[k] == 0).all()) and bool((hr[k] == 0).all()), k
    assert torch.equal(prev[1].view(torch.int32), prev0[1].view(torch.int32))
    assert torch.equal(hr[1].view(torch.int32), hr0[1].view(torch.int32))
    _bits(lr.cpu().numpy(), _decode_ref(frames, layout, 'bt601-full'))


# ------------------------------------------------------------------------------------------------ encode kernel
def _encode(layout, color, src, out_offset=0):
    """tg_rgb_to_yuv of src (uint8 NHWC numpy for 8 bit, fp32 NCHW numpy for 10 bit) into an output placed
    out_offset bytes past 16 inside a 0xAB guard band; returns (words, guard intact)."""
    ten = C.depth_of(layout) == 10
    n, H, W = (src.shape[0], src.shape[2], src.shape[3]) if ten else src.shape[:3]
    shape = (n, *C.frame_shape(layout, H, W))
    nout = int(np.prod(shape)) * (2 if ten else 1)
    buf, region = _placed(nout, out_offset)
    out = (region.view(torch.uint16) if ten else region).view(shape)
    s = torch.from_numpy(np.ascontiguousarray(src)).to(DEV)
    ops.rgb_to_yuv(layout, color, **({'rgb_f32': s} if ten else {'rgb_u8': s}), out=out)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    guard = bool((b[:out_offset] == GUARD).all() and (b[out_offset + nout:] == GUARD).all())
    return b[out_offset:out_offset + nout].view(np.uint16 if ten else np.uint8).reshape(shape), guard


@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('layout', NEW8)
def test_kernel_encode_every_rgb_triple(layout, color):
    """2^24 pixels, each block's top-left pixel a different RGB triple and its right neighbour 255 - that triple
    (8 frames of 1024 x 8192)."""
    rgb = np.stack([Y8.rgb_triples_pattern(r, 512) for r in range(0, 4096, 512)])
    got, guard = _encode(layout, color, rgb)
    assert guard
    for k in range(rgb.shape[0]):
        want = C.rgb_to_yuv(rgb[k], layout, color)
        assert np.array_equal(got[k], want), (k, int((got[k] != want).sum()))


@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('layout', NEW8)
@pytest.mark.parametrize('n,H,W,off', [(3, 37, 54, 4), (2, 3, 1030, 8), (1, 1, 2, 0), (2, 5, 513, 12)])
def test_kernel_encode_8bit_ragged(layout, color, n, H, W, off):
    if layout in C.LAYOUTS_422:
        W += W % 2
    elif off:
        off += 1                                          # planar bytes: odd offsets too
    rgb = np.random.default_rng(5000 + H + W + off).integers(0, 256, size=(n, H, W, 3), dtype=np.uint8)
    got, guard = _encode(layout, color, rgb, off)
    assert guard and np.array_equal(got, C.rgb_to_yuv(rgb, layout, color))


def _f32_frames(n, H, W, seed):
    """fp32 NCHW frames with negatives, values above 1 and exact .5 ties of x * 1023."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-0.2, 1.2, size=(n, 3, H, W)).astype(np.float32)
    ties = (rng.integers(0, 1023, size=x.shape).astype(np.float32) + np.float32(0.5)) / np.float32(1023.0)
    pick = rng.random(x.shape) < 0.3
    x[pick] = ties[pick]
    return x


@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('n,H,W,off', [(2, 37, 54, 0), (1, 3, 523, 6), (2, 536, 1280, 2), (1, 1, 1, 14)])
def test_kernel_encode_i444_10_from_fp32(color, n, H, W, off):
    x = _f32_frames(n, H, W, 6000 + H + W + off)
    got, guard = _encode('i444_10', color, x, off)
    assert guard
    assert np.array_equal(got, C.rgb_f32_to_yuv(x.transpose(0, 2, 3, 1), 'i444_10', color))


# ------------------------------------------------------------------------------------------------ streams
def _clips_u8(seed, n, t, c, h, w):
    clips = [synthetic.make_clip(seed + k, t, c, h, w, shift=1 + k).numpy() for k in range(n)]
    return np.ascontiguousarray((np.rint(np.stack(clips) * 255.0)).astype(np.uint8).transpose(0, 1, 3, 4, 2))


def _cut_clips_u8(h, w):
    """uint8 RGB [2,10,h,w,3]: slot 0 cuts from one clip to another at frame 6, slot 1 is one clip."""
    a = np.concatenate([synthetic.make_clip(1, 6, 3, h, w).numpy(), synthetic.make_clip(2, 4, 3, h, w).numpy()])
    b = synthetic.make_clip(3, 10, 3, h, w).numpy()
    return np.ascontiguousarray((np.rint(np.stack([a, b]) * 255.0)).astype(np.uint8).transpose(0, 1, 3, 4, 2))


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


def _hr_loop(net, rgb_f32, resets):
    """fp32 HR frames [n,t,3,H,W] (on the device) of a loop of net.step over lr [n,t,3,h,w], zero state at frame 0
    and for slot k at frame i when (k, i) in resets."""
    n, t = rgb_f32.shape[:2]
    lr = torch.from_numpy(rgb_f32).to(DEV)
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


def _nhwc(hr):
    return hr.permute(0, 1, 3, 4, 2).cpu().numpy()


def _dec(frames, layout, color):
    """(RGB codes [n,t,h,w,3], the stream's fp32 input [n,t,3,h,w]) of YUV frames [n,t,...]."""
    rgb = C.yuv_to_rgb(frames, layout, color)
    scale = np.float32(1023.0 if C.depth_of(layout) == 10 else 255.0)
    return rgb, np.ascontiguousarray((rgb.astype(np.float32) / scale).transpose(0, 1, 4, 2, 3))


GEOMS = {'bd4': (134, 320), 'bi2': (37, 54)}       # bench.py's bd4 frame; an odd height for bi2


@pytest.mark.parametrize('geom', ['bd4', 'bi2'])
def test_chunked_pushes_match_oracle(geom, bd4_net, bi2_net):
    """n=2 clips of 10 frames pushed as [1,4,2,3] with slot 1 restarting at frame 5, host and device I/O: every new
    layout in (against the RGB / fp32 stream of its decode) and out (against the encode of the RGB stream's bytes or
    of the fp32 HR frames of a device FRNet.step loop)."""
    net = bd4_net if geom == 'bd4' else bi2_net
    h, w = GEOMS[geom]
    u8 = _clips_u8(81, 2, 10, 3, h, w)
    chunks, resets = [1, 4, 2, 3], [None, None, [False, True], None]
    reset_at = {(1, 5)}
    rgb10 = np.rint(u8.astype(np.float64) * (1023.0 / 255.0)).astype(np.int64)
    colors = {'yuy2': 'bt601', 'uyvy': 'bt709', 'i444': 'bt709-full', 'i444_10': 'bt601-full'}
    for out in ('host', 'device'):
        for layout in NEW8:
            color = colors[layout]
            frames = C.rgb_to_yuv(u8, layout, color)
            rgb_in, _ = _dec(frames, layout, color)
            ref = _push(net.stream(2, h, w, device=DEV), rgb_in, chunks, resets)
            # in: the RGB stream of the decoded frames
            s = net.stream(2, h, w, device=DEV, input=layout, in_color=color)
            got = _push(s, frames, chunks, resets, out)
            s.close()
            assert np.array_equal(got, ref), (layout, out)
            # in and out: the encode of that RGB output
            s = net.stream(2, h, w, device=DEV, input=layout, in_color=color, out_format=layout, out_color=color)
            got = _push(s, frames, chunks, resets, out)
            s.close()
            want = C.rgb_to_yuv(ref, layout, color)
            assert got.dtype == np.uint8 and np.array_equal(got, want), (layout, out, int((got != want).sum()))
        # I444_10 in and out: the 10-bit encode of the fp32 HR frames of a step loop over decode / 1023
        color = colors['i444_10']
        frames = C.rgb_to_yuv(rgb10, 'i444_10', color)
        _, f32 = _dec(frames, 'i444_10', color)
        s = net.stream(2, h, w, device=DEV, input='i444_10', in_color=color, out_format='i444_10', out_color=color)
        got = _push(s, frames, chunks, resets, out)
        s.close()
        want = C.rgb_f32_to_yuv(_nhwc(_hr_loop(net, f32, reset_at)), 'i444_10', color)
        assert got.dtype == np.uint16 and np.array_equal(got, want), (out, int((got != want).sum()))
        # I444_10 in, RGB out: the float32 stream of decode / 1023
        s = net.stream(2, h, w, device=DEV, input='i444_10', in_color=color)
        got = _push(s, frames, chunks, resets, out)
        s.close()
        assert np.array_equal(got, _push(net.stream(2, h, w, device=DEV, input='float32'), f32, chunks, resets)), out


def test_resized_output(bi2_net):
    """out_size with 4:2:2 / 4:4:4 output: the encode of the resized uint8 RGB stream (8 bit), or of the resize
    kernel's fp32 output of a step loop's HR frames (I444_10); odd Ho (and odd Wo for 4:4:4)."""
    net, (h, w) = bi2_net, GEOMS['bi2']
    u8 = _clips_u8(91, 2, 6, 3, h, w)
    chunks, resets = [2, 1, 3], [None, [True, False], None]
    frames = C.rgb_to_yuv(u8, 'uyvy', 'bt709')
    rgb_in, f32 = _dec(frames, 'uyvy', 'bt709')
    for layout, size in (('yuy2', (61, 130)), ('uyvy', (75, 108)), ('i444', (61, 131))):
        ref = _push(net.stream(2, h, w, device=DEV, out_size=size), rgb_in, chunks, resets)
        s = net.stream(2, h, w, device=DEV, input='uyvy', in_color='bt709', out_format=layout, out_color='bt709',
                       out_size=size)
        got = _push(s, frames, chunks, resets)
        s.close()
        assert got.shape == (2, 6, *C.frame_shape(layout, *size)) and np.array_equal(
            got, C.rgb_to_yuv(ref, layout, 'bt709')), layout
    size = (61, 131)
    hr = _hr_loop(net, f32, {(0, 2)})
    tabs = [tuple(t.to(DEV) for t in ops.resample_table(a, b, 'bicubic')) for a, b in zip(hr.shape[-2:], size)]
    rs = torch.stack([ops.resample(hr[:, i].contiguous(), *tabs, out_f32=torch.empty(2, 3, *size, device=DEV))
                      for i in range(hr.shape[1])], dim=1)
    s = net.stream(2, h, w, device=DEV, input='uyvy', in_color='bt709', out_format='i444_10', out_size=size)
    got = _push(s, frames, chunks, resets)
    s.close()
    assert np.array_equal(got, C.rgb_f32_to_yuv(_nhwc(rs), 'i444_10', 'bt601'))


def test_scene_cuts_and_single_frame_pushes(bi2_net):
    """scene_cut= with YUY2 in / UYVY out and I444 in / I444 out, pushed one frame at a time: the same cuts and
    scores as the uint8 stream of the decoded frames, and the encode of its output."""
    net, (h, w) = bi2_net, GEOMS['bi2']
    u8 = _cut_clips_u8(h, w)
    chunks = [1] * 10
    for lin, lout, color in (('yuy2', 'uyvy', 'bt601'), ('i444', 'i444', 'bt709')):
        frames = C.rgb_to_yuv(u8, lin, color)
        rgb_in, _ = _dec(frames, lin, color)
        ref_s = net.stream(2, h, w, device=DEV, scene_cut=THR)
        ref, ref_cuts = [], []
        for i in range(10):
            ref.append(ref_s.push(rgb_in[:, i:i + 1]))
            ref_cuts.append(ref_s.last_cuts)
        ref = np.concatenate(ref, axis=1)
        assert np.concatenate(ref_cuts, axis=1)[0].any()                       # the cut is detected
        s = net.stream(2, h, w, device=DEV, scene_cut=THR, input=lin, in_color=color, out_format=lout,
                       out_color=color)
        got, cuts = [], []
        for i, k in enumerate(chunks):
            got.append(s.push(frames[:, i:i + k]))
            cuts.append(s.last_cuts)
        s.close()
        assert np.array_equal(np.concatenate(cuts, axis=1), np.concatenate(ref_cuts, axis=1)), lin
        assert np.array_equal(np.concatenate(got, axis=1), C.rgb_to_yuv(ref, lout, color)), lin


def test_single_slot_three_dim_frames(bi2_net):
    net, (h, w) = bi2_net, GEOMS['bi2']
    u8 = _clips_u8(95, 1, 3, 3, h, w)
    frames = C.rgb_to_yuv(u8, 'yuy2', 'bt601')[0]                              # [k, h, 2w]
    ref = net.stream(1, h, w, device=DEV).push(C.yuv_to_rgb(frames, 'yuy2')[None])
    got = net.stream(1, h, w, device=DEV, input='yuy2', out_format='yuy2').push(frames)
    assert got.shape == (1, 3, 2 * h, 4 * w) and np.array_equal(got, C.rgb_to_yuv(ref, 'yuy2'))
