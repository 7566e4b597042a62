"""pytest -m gpu: BT.601 / BT.709, limited / full range and 10-bit (P010, I420_10) frame I/O of streamed inference --
the kernels tg_stream_frame_in_yuv and tg_rgb_to_yuv and FRNet.stream(in_color=, out_color=, input='p010', ...).

The specification is oracle/yuv_color.py (checked on the CPU by tests/test_yuv_color_oracle_cpu.py); every kernel
output below equals it bit for bit.  Every output buffer is filled with NaN or 0xAB first."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import yuv_color as C              # noqa: E402
from oracle import yuv_oracle as Y8            # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
BD4 = dict(scale=4, degradation='BD', c=3, h=134, w=320)      # bench.py's bd4 frame
BI2 = dict(scale=2, degradation='BI', c=3, h=36, w=52)
GUARD = 0xAB


def _net(scale, degradation):
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def bd4_net():
    return _net(4, 'BD')


def _placed(nbytes, offset):
    """A uint8 device buffer of 0xAB with `offset` guard bytes before and 64 after a region; returns (buf, region)."""
    buf = torch.full((offset + nbytes + 64,), GUARD, dtype=torch.uint8, device=DEV)
    return buf, buf[offset:offset + nbytes]


def _to_dev(frames, offset=0):
    """numpy uint8 / uint16 frames [n,3h/2,w] -> a device tensor of the same dtype `offset` bytes past 16."""
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


# ------------------------------------------------------------------------------------------------ decode kernel
@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('layout', C.LAYOUTS)
def test_kernel_decode_every_sample(layout, color):
    """8 bit: the 4096x4096 frame with every (Y, U, V) triple; 10 bit: every triple of the dense sample, with junk in
    P010's low bits and I420_10 words above 1023."""
    if C.depth_of(layout) == 8:
        frames = C.yuv_triples_pattern(layout)[None]
        h = w = 4096
    else:
        frames, h, w = C.yuv10_pattern(layout)
    lr, _, _ = _decode(_to_dev(frames), layout, color, frames.shape[0], h, w)
    _bits(lr.cpu().numpy(), _decode_ref(frames, layout, color))


@pytest.mark.parametrize('layout', C.LAYOUTS)
@pytest.mark.parametrize('n,h,w,offset', [(3, 38, 54, 6), (2, 6, 300, 14), (1, 4, 520, 2), (2, 2, 2, 0)])
def test_kernel_decode_ragged_misaligned(layout, n, h, w, offset):
    """Rows and planes not multiples of 16 bytes, more than one tile wide, sources at word-aligned offsets past a
    16-byte boundary (odd offsets too for uint8); lr_prev / hr_prev untouched without a mask."""
    rng = np.random.default_rng(3000 + n * h + w + offset)
    dt = C.word_dtype(layout)
    frames = rng.integers(0, np.iinfo(dt).max + 1, size=(n, 3 * h // 2, w)).astype(dt)
    off = offset + (1 if dt == np.uint8 else 0)
    lr, prev, hr = _decode(_to_dev(frames, off), layout, 'bt709', n, h, w, s=4)
    _bits(lr.cpu().numpy(), _decode_ref(frames, layout, 'bt709'))
    assert bool((prev == 3.0).all()) and bool((hr == 5.0).all())


@pytest.mark.parametrize('layout', ['p010', 'i420_10', 'nv12'])
def test_kernel_decode_reset_zeroes_flagged_slots_only(layout):
    n, h, w, s = 3, 38, 54, 4
    g = torch.Generator(device=DEV).manual_seed(9)
    prev = torch.rand((n, 3, h, w), generator=g, device=DEV) + 1.0
    hr = torch.rand((n, 3, s * h, s * w), generator=g, device=DEV) + 1.0
    prev0, hr0 = prev.clone(), hr.clone()
    frames = np.random.default_rng(5).integers(0, 1 << 16, size=(n, 3 * h // 2, w)).astype(C.word_dtype(layout))
    mask = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    lr, prev, hr = _decode(_to_dev(frames), layout, 'bt601-full', n, h, w, s, reset=mask, prev=prev, hr=hr)
    for k in (0, 2):
        assert bool((prev[k] == 0).all()) and bool((hr[k] == 0).all()), k
    assert torch.equal(prev[1].view(torch.int32), prev0[1].view(torch.int32))
    assert torch.equal(hr[1].view(torch.int32), hr0[1].view(torch.int32))
    _bits(lr.cpu().numpy(), _decode_ref(frames, layout, 'bt601-full'))


@pytest.mark.parametrize('layout', Y8.LAYOUTS)
def test_default_format_is_the_old_decode(layout):
    rng = np.random.default_rng(77)
    frames = rng.integers(0, 256, size=(2, 57, 76), dtype=np.uint8)
    new, _, _ = _decode(_to_dev(frames), layout, 'bt601', 2, 38, 76)
    old = torch.full_like(new, float('nan'))
    ops.stream_frame_in_yuv420(_to_dev(frames), layout, None, old, torch.empty_like(old),
                               torch.empty(2, 3, 76, 152, device=DEV), 2)
    torch.cuda.synchronize()
    assert torch.equal(new.view(torch.int32), old.view(torch.int32))


# ------------------------------------------------------------------------------------------------ encode kernel
def _encode(layout, color, src, out_offset=0):
    """tg_rgb_to_yuv of src (uint8 NHWC numpy for 8 bit, fp32 NCHW numpy for 10 bit) into an output placed
    out_offset bytes past 16 inside a 0xAB guard band; returns (words, guard intact)."""
    ten = C.depth_of(layout) == 10
    n, H, W = (src.shape[0], src.shape[2], src.shape[3]) if ten else src.shape[:3]
    wb = 2 if ten else 1
    nout = n * 3 * H // 2 * W * wb
    buf, region = _placed(nout, out_offset)
    out = (region.view(torch.uint16) if ten else region).view(n, 3 * H // 2, W)
    s = torch.from_numpy(np.ascontiguousarray(src)).to(DEV)
    ops.rgb_to_yuv(layout, color, **({'rgb_f32': s} if ten else {'rgb_u8': s}), out=out)
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    guard = bool((b[:out_offset] == GUARD).all() and (b[out_offset + nout:] == GUARD).all())
    words = b[out_offset:out_offset + nout].view(np.uint16 if ten else np.uint8).reshape(n, 3 * H // 2, W)
    return words, guard


@pytest.mark.parametrize('color', ['bt709', 'bt601-full', 'bt709-full'])
def test_kernel_encode_every_rgb_triple(color):
    """2^24 blocks, each with a different RGB triple as its top-left pixel (8 frames of 1024 x 8192)."""
    rgb = np.stack([Y8.rgb_triples_pattern(r, 512) for r in range(0, 4096, 512)])
    layout = 'nv12' if color != 'bt601-full' else 'i420'
    got, guard = _encode(layout, color, rgb)
    assert guard
    for k in range(rgb.shape[0]):
        want = C.rgb_to_yuv(rgb[k], layout, color)
        assert np.array_equal(got[k], want), (k, int((got[k] != want).sum()))


def _f32_frames(n, H, W, seed):
    """fp32 NCHW frames with negatives, values above 1 and exact .5 ties of x * 1023."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-0.2, 1.2, size=(n, 3, H, W)).astype(np.float32)
    ties = (rng.integers(0, 1023, size=x.shape).astype(np.float32) + np.float32(0.5)) / np.float32(1023.0)
    pick = rng.random(x.shape) < 0.3
    x[pick] = ties[pick]
    return x


@pytest.mark.parametrize('layout', ['p010', 'i420_10'])
@pytest.mark.parametrize('color', C.COLORS)
@pytest.mark.parametrize('n,H,W,off', [(2, 38, 54, 0), (1, 4, 522, 6), (2, 536, 1280, 2), (1, 2, 2, 14)])
def test_kernel_encode_10bit_from_fp32(layout, color, n, H, W, off):
    x = _f32_frames(n, H, W, 4000 + H + W + off)
    got, guard = _encode(layout, color, x, off)
    assert guard
    want = C.rgb_f32_to_yuv(x.transpose(0, 2, 3, 1), layout, color)
    assert np.array_equal(got, want), int((got != want).sum())


@pytest.mark.parametrize('layout', Y8.LAYOUTS)
@pytest.mark.parametrize('n,H,W,off', [(3, 38, 54, 7), (2, 4, 522, 9), (1, 10, 1030, 3)])
def test_kernel_encode_8bit_ragged_and_default_is_old(layout, n, H, W, off):
    rgb = np.random.default_rng(5000 + H + W).integers(0, 256, size=(n, H, W, 3), dtype=np.uint8)
    got, guard = _encode(layout, 'bt709-full', rgb, off)
    assert guard and np.array_equal(got, C.rgb_to_yuv(rgb, layout, 'bt709-full'))
    new, guard = _encode(layout, 'bt601', rgb, off)
    old = ops.rgb_u8_to_yuv420(torch.from_numpy(rgb).to(DEV), layout).cpu().numpy()
    assert guard and np.array_equal(new, old)


# ------------------------------------------------------------------------------------------------ streams
def _clips_u8(seed, n, t, c, h, w):
    clips = [synthetic.make_clip(seed + k, t, c, h, w, shift=1 + k).numpy() for k in range(n)]
    return np.ascontiguousarray((np.rint(np.stack(clips) * 255.0)).astype(np.uint8).transpose(0, 1, 3, 4, 2))


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
    """fp32 HR frames [n,t,H,W,3] of a device loop of net.step over lr [n,t,3,h,w] (fp32), zero state at frame 0 and
    for slot k at frame i when (k, i) in resets."""
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
            outs.append(hr.permute(0, 2, 3, 1).cpu().numpy())
            lr_prev, hr_prev = lr[:, i].contiguous(), hr
    return np.stack(outs, axis=1)


@pytest.mark.parametrize('geom', [BD4, BI2], ids=['bd4', 'bi2'])
def test_chunked_color_pushes_match_oracle(geom, bd4_net):
    """n=2 clips of 10 frames pushed as [1,4,2,3] with slot 1 restarting at frame 5 (the third chunk), host and
    device I/O: P010/BT.709 -> P010/BT.709, NV12/BT.601 -> NV12/BT.709, I420_10/full -> RGB, RGB -> P010."""
    net = bd4_net if geom is BD4 else _net(geom['scale'], geom['degradation'])
    c, h, w = geom['c'], geom['h'], geom['w']
    u8 = _clips_u8(61, 2, 10, c, h, w)
    chunks, resets = [1, 4, 2, 3], [None, None, [False, True], None]
    reset_at = {(1, 5)}
    rgb10 = np.rint(u8.astype(np.float64) * (1023.0 / 255.0)).astype(np.int64)
    p010 = C.rgb_to_yuv(rgb10, 'p010', 'bt709')
    i42010 = C.rgb_to_yuv(rgb10, 'i420_10', 'bt709-full')
    nv12 = C.rgb_to_yuv(u8, 'nv12', 'bt601')

    def dec(frames, layout, color):
        rgb = C.yuv_to_rgb(frames, layout, color)
        scale = np.float32(1023.0 if C.depth_of(layout) == 10 else 255.0)
        return rgb, np.ascontiguousarray((rgb.astype(np.float32) / scale).transpose(0, 1, 4, 2, 3))

    def rgb_stream(rgb_u8):
        return _push(net.stream(2, h, w, device=DEV), rgb_u8, chunks, resets)

    for out in ('host', 'device'):
        # P010 / BT.709 -> P010 / BT.709: the oracle's encode of the fp32 HR frames of the decoded input
        _, f32 = dec(p010, 'p010', 'bt709')
        s = net.stream(2, h, w, device=DEV, input='p010', out_format='p010', in_color='bt709', out_color='bt709')
        got = _push(s, p010, chunks, resets, out)
        want = C.rgb_f32_to_yuv(_hr_loop(net, f32, reset_at), 'p010', 'bt709')
        assert got.dtype == np.uint16 and np.array_equal(got, want), (out, int((got != want).sum()))
        s.close()
        # NV12 / BT.601 -> NV12 / BT.709: the oracle's BT.709 encode of the RGB stream's bytes
        rgb_in, _ = dec(nv12, 'nv12', 'bt601')
        ref = rgb_stream(rgb_in)
        s = net.stream(2, h, w, device=DEV, input='nv12', out_format='nv12', out_color='bt709')
        got = _push(s, nv12, chunks, resets, out)
        assert np.array_equal(got, C.rgb_to_yuv(ref, 'nv12', 'bt709')), out
        s.close()
        # I420_10 / full -> RGB: the uint8 output of the same step as the fp32 input of the decoded frames
        _, f32 = dec(i42010, 'i420_10', 'bt709-full')
        s = net.stream(2, h, w, device=DEV, input='i420_10', in_color='bt709-full')
        got = _push(s, i42010, chunks, resets, out)
        want = _push(net.stream(2, h, w, device=DEV, input='float32'), f32, chunks, resets)
        assert np.array_equal(got, want), out
        s.close()
        # RGB -> P010 / BT.601 limited
        f32 = np.ascontiguousarray((u8.astype(np.float32) / np.float32(255.0)).transpose(0, 1, 4, 2, 3))
        s = net.stream(2, h, w, device=DEV, out_format='p010')
        got = _push(s, u8, chunks, resets, out)
        want = C.rgb_f32_to_yuv(_hr_loop(net, f32, reset_at), 'p010', 'bt601')
        assert np.array_equal(got, want), (out, int((got != want).sum()))
        s.close()
