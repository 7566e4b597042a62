"""pytest -m gpu: YUV 4:2:0 (NV12 / I420) frame I/O of streamed inference -- the kernels
tg_stream_frame_in_yuv420 and tg_rgb_u8_to_yuv420 and FRNet.stream(input=, out_format=).

The specification is oracle/yuv_oracle.py (cv2.cvtColor restated in integer numpy, pinned to cv2 by
tests/test_yuv_oracle_cpu.py):
- the decode kernel gives the oracle's RGB / 255 bit for bit for every (Y, U, V) triple and for ragged,
  misaligned frames, and its reset zeroes only flagged slots;
- the encode kernel gives the oracle's bytes for every RGB triple as the top-left pixel of a block and for
  widths that are not a multiple of 16, and writes no byte outside its output;
- a YUV stream pushed in chunks gives the oracle conversions around the RGB stream (itself pinned to
  infer_sequence), with slot resets and with device input and output.
Every kernel output buffer is filled with NaN or 0xAB first."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import yuv_oracle as Y             # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
BD4 = dict(scale=4, degradation='BD', c=3, h=134, w=320)      # bench.py's bd4 frame
BI2 = dict(scale=2, degradation='BI', c=3, h=36, w=52)
GUARD = 0xAB


def _net(scale, degradation):
    """bench.make_params() weights (seed 0, gain 1) for the given workload."""
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def bd4_net():
    return _net(4, 'BD')


def _clips_u8(seed, n, t, c, h, w):
    """n different smooth clips as uint8 [n,t,h,w,c] (numpy)."""
    clips = [synthetic.make_clip(seed + k, t, c, h, w, shift=1 + k).numpy() for k in range(n)]
    return np.ascontiguousarray((np.rint(np.stack(clips) * 255.0)).astype(np.uint8).transpose(0, 1, 3, 4, 2))


def _push_chunks(stream, frames, chunks, **kw):
    out, i = [], 0
    for k in chunks:
        o = stream.push(frames[:, i:i + k], **kw)
        out.append(o.cpu().numpy() if isinstance(o, torch.Tensor) else o)
        i += k
    assert i == frames.shape[1]
    return np.concatenate(out, axis=1)


def _placed(nbytes, offset, fill=GUARD):
    """A uint8 device buffer with `offset` guard bytes before and 64 after a region of nbytes; returns (buf, region)."""
    buf = torch.full((offset + nbytes + 64,), fill, dtype=torch.uint8, device=DEV)
    return buf, buf[offset:offset + nbytes]


def _assert_bits(got, want):
    assert got.dtype == np.float32 and got.shape == want.shape
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), (int(bad.sum()), np.argwhere(bad)[:4].tolist())


# ------------------------------------------------------------------------------------------------ decode kernel
def _decode_ref(frames, layout):
    """oracle RGB / 255 as numpy float32 [n,3,h,w] (the reference loader's division)."""
    return np.ascontiguousarray(Y.yuv420_to_rgb(frames, layout).astype(np.float32).transpose(0, 3, 1, 2)
                                / np.float32(255.0))


@pytest.mark.parametrize('layout', Y.LAYOUTS)
def test_kernel_decode_every_yuv_triple(layout):
    """The 4096x4096 frame that holds each of the 2^24 (Y, U, V) triples once."""
    frame = Y.yuv_triples_pattern(layout)[None]
    n, h, w, s = 1, 4096, 4096, 2
    yuv = torch.from_numpy(frame).to(DEV)
    lr = torch.full((n, 3, h, w), float('nan'), device=DEV)
    prev = torch.empty((n, 3, h, w), device=DEV)
    hr = torch.empty((n, 3, s * h, s * w), device=DEV)
    ops.stream_frame_in_yuv420(yuv, layout, None, lr, prev, hr, s)
    torch.cuda.synchronize()
    _assert_bits(lr.cpu().numpy(), _decode_ref(frame, layout))


@pytest.mark.parametrize('layout', Y.LAYOUTS)
@pytest.mark.parametrize('n,h,w,offset', [(3, 38, 54, 5), (2, 6, 300, 13), (1, 4, 520, 3), (2, 2, 2, 0),
                                          (1, 38, 54, 0)])
def test_kernel_decode_ragged_misaligned(layout, n, h, w, offset):
    """Random frames whose rows and planes are not multiples of 16 bytes, more than one 256-pixel tile wide, read
    from a source `offset` bytes past a 16-byte boundary; without a mask lr_prev / hr_prev are untouched."""
    s = 4
    rng = np.random.default_rng(1000 + n * h + w + offset)
    frames = rng.integers(0, 256, size=(n, 3 * h // 2, w), dtype=np.uint8)
    _, src = _placed(frames.size, offset)
    src.copy_(torch.from_numpy(frames).reshape(-1))
    lr = torch.full((n, 3, h, w), float('nan'), device=DEV)
    prev = torch.full_like(lr, 3.0)
    hr = torch.full((n, 3, s * h, s * w), 5.0, device=DEV)
    ops.stream_frame_in_yuv420(src.view(n, 3 * h // 2, w), layout, None, lr, prev, hr, s)
    torch.cuda.synchronize()
    _assert_bits(lr.cpu().numpy(), _decode_ref(frames, layout))
    assert bool((prev == 3.0).all()) and bool((hr == 5.0).all())


@pytest.mark.parametrize('layout', Y.LAYOUTS)
@pytest.mark.parametrize('with_frames', [True, False], ids=['decode_and_reset', 'reset_only'])
def test_kernel_decode_reset_zeroes_flagged_slots_only(layout, with_frames):
    n, h, w, s = 3, 38, 54, 4         # a slot of lr_prev is 6156 floats: slot starts are not all 16-byte aligned
    g = torch.Generator(device=DEV).manual_seed(9)
    lr = torch.full((n, 3, h, w), float('nan'), device=DEV)
    prev = torch.rand((n, 3, h, w), generator=g, device=DEV) + 1.0
    hr = torch.rand((n, 3, s * h, s * w), generator=g, device=DEV) + 1.0
    prev0, hr0 = prev.clone(), hr.clone()
    yuv = (torch.randint(0, 256, (n, 3 * h // 2, w), generator=g, device=DEV, dtype=torch.uint8)
           if with_frames else None)
    mask = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    ops.stream_frame_in_yuv420(yuv, layout, mask, lr, prev, hr, s)
    torch.cuda.synchronize()
    for k in (0, 2):
        assert bool((prev[k] == 0).all()) and bool((hr[k] == 0).all()), k
    assert torch.equal(prev[1].view(torch.int32), prev0[1].view(torch.int32))
    assert torch.equal(hr[1].view(torch.int32), hr0[1].view(torch.int32))
    if with_frames:
        _assert_bits(lr.cpu().numpy(), _decode_ref(yuv.cpu().numpy(), layout))
    else:
        assert bool(torch.isnan(lr).all())                                  # in = NULL: lr_curr is not written
    mask.zero_()
    ops.stream_frame_in_yuv420(yuv, layout, mask, lr, prev0, hr0, s)       # an all-zero mask writes nothing
    torch.cuda.synchronize()
    assert bool((prev0 > 0).all()) and bool((hr0 > 0).all())


# ------------------------------------------------------------------------------------------------ encode kernel
def _encode(rgb_np, layout, in_offset=0, out_offset=0):
    """Run tg_rgb_u8_to_yuv420 on rgb [n,H,W,3] placed `in_offset` bytes past a 16-byte boundary into an output
    `out_offset` bytes past one, inside a 0xAB guard band; returns (output, guard bytes intact)."""
    n, H, W, _ = rgb_np.shape
    _, src = _placed(rgb_np.size, in_offset)
    src.copy_(torch.from_numpy(rgb_np).reshape(-1))
    nout = n * 3 * H // 2 * W
    buf, dst = _placed(nout, out_offset)
    ops.rgb_u8_to_yuv420(src.view(n, H, W, 3), layout, out=dst.view(n, 3 * H // 2, W))
    torch.cuda.synchronize()
    b = buf.cpu().numpy()
    guard_ok = bool((b[:out_offset] == GUARD).all() and (b[out_offset + nout:] == GUARD).all())
    return b[out_offset:out_offset + nout].reshape(n, 3 * H // 2, W), guard_ok


@pytest.mark.parametrize('layout', Y.LAYOUTS)
def test_kernel_encode_every_rgb_triple(layout):
    """2^24 blocks, each with a different RGB triple as its top-left pixel (and other values in the rest), as 8
    frames of 1024 x 8192."""
    rgb = np.stack([Y.rgb_triples_pattern(r, 512) for r in range(0, 4096, 512)])      # [8,1024,8192,3]
    got, guard_ok = _encode(rgb, layout)
    assert guard_ok
    for k in range(rgb.shape[0]):
        want = Y.rgb_to_yuv420(rgb[k], layout)
        assert np.array_equal(got[k], want), (k, int((got[k] != want).sum()))


@pytest.mark.parametrize('layout', Y.LAYOUTS)
@pytest.mark.parametrize('n,H,W,in_off,out_off', [(3, 38, 54, 0, 0), (3, 38, 54, 5, 7), (2, 4, 522, 1, 9),
                                                  (1, 2, 2, 3, 15), (2, 536, 1280, 0, 0), (1, 10, 1030, 0, 3)])
def test_kernel_encode_ragged_widths_and_guard_band(layout, n, H, W, in_off, out_off):
    """W not a multiple of 16 (and not of the 256-pixel tile), misaligned source and destination; no byte
    outside [n,3H/2,W] written."""
    rng = np.random.default_rng(2000 + n * H + W + in_off)
    rgb = rng.integers(0, 256, size=(n, H, W, 3), dtype=np.uint8)
    got, guard_ok = _encode(rgb, layout, in_off, out_off)
    assert guard_ok
    want = Y.rgb_to_yuv420(rgb, layout)
    assert np.array_equal(got, want), int((got != want).sum())


# ------------------------------------------------------------------------------------------------ streams
def _yuv_clip(u8, layout):
    """uint8 [n,t,h,w,3] -> (YUV frames [n,t,3h/2,w] of the oracle, the RGB frames they decode to)."""
    yuv = Y.rgb_to_yuv420(u8, layout)
    return yuv, Y.yuv420_to_rgb(yuv, layout)


@pytest.mark.parametrize('geom', [BD4, BI2], ids=['bd4', 'bi2'])
def test_chunked_yuv_push_matches_oracle_around_rgb_stream(geom, bd4_net):
    """n=2 clips of 10 frames pushed as chunks [1,4,2,3]: NV12 -> NV12, I420 -> I420, NV12 -> RGB and RGB -> NV12
    give the oracle's conversions around the RGB stream of the decoded frames."""
    net = bd4_net if geom is BD4 else _net(geom['scale'], geom['degradation'])
    c, h, w = geom['c'], geom['h'], geom['w']
    u8 = _clips_u8(13, 2, 10, c, h, w)
    chunks = [1, 4, 2, 3]
    nv12, rgb_in = _yuv_clip(u8, 'nv12')
    i420, rgb_in_i420 = _yuv_clip(u8, 'i420')
    assert np.array_equal(rgb_in, rgb_in_i420)              # the same planes, laid out twice
    ref = _push_chunks(net.stream(2, h, w, device=DEV), rgb_in, chunks)                  # [n,t,H,W,3]
    assert np.array_equal(ref, net.infer_sequence(
        torch.from_numpy(rgb_in.astype(np.float32) / np.float32(255.0)).permute(0, 1, 4, 2, 3).contiguous(), DEV))
    cases = [('nv12', 'nv12', nv12, Y.rgb_to_yuv420(ref, 'nv12')),
             ('i420', 'i420', i420, Y.rgb_to_yuv420(ref, 'i420')),
             ('nv12', 'rgb', nv12, ref),
             ('uint8', 'nv12', rgb_in, Y.rgb_to_yuv420(ref, 'nv12'))]
    for inp, fmt, frames, want in cases:
        s = net.stream(2, h, w, device=DEV, input=inp, out_format=fmt)
        got = _push_chunks(s, torch.from_numpy(frames), chunks)
        assert got.shape == want.shape and got.dtype == np.uint8, (inp, fmt)
        assert np.array_equal(got, want), (inp, fmt, int((got != want).sum()))
        s.close()


def test_float32_input_with_i420_output():
    net = _net(BI2['scale'], BI2['degradation'])
    c, h, w = BI2['c'], BI2['h'], BI2['w']
    u8 = _clips_u8(17, 2, 4, c, h, w)
    f32 = torch.from_numpy(u8.astype(np.float32) / np.float32(255.0)).permute(0, 1, 4, 2, 3).contiguous()
    ref = _push_chunks(net.stream(2, h, w, device=DEV), u8, [4])
    got = _push_chunks(net.stream(2, h, w, device=DEV, input='float32', out_format='i420'), f32, [3, 1])
    assert np.array_equal(got, Y.rgb_to_yuv420(ref, 'i420'))


def test_nv12_slot_reset_restarts_one_slot(bd4_net):
    """Slot 1 switches from video B to video C at frame 5 while slot 0 plays video A throughout, NV12 in and out:
    the oracle around the RGB stream with the same restart."""
    net = bd4_net
    c, h, w = BD4['c'], BD4['h'], BD4['w']
    a, b, cc = (_clips_u8(seed, 1, 10, c, h, w) for seed in (23, 33, 43))
    u8 = np.concatenate([a, np.concatenate([b[:, :5], cc[:, :5]], axis=1)], axis=0)      # [2,10,h,w,c]
    nv12, rgb_in = _yuv_clip(u8, 'nv12')
    r = net.stream(2, h, w, device=DEV)
    ref = np.concatenate([r.push(rgb_in[:, :3]), r.push(rgb_in[:, 3:5]), r.push(rgb_in[:, 5:], reset=[False, True])],
                         axis=1)
    fresh = net.infer_sequence(torch.from_numpy(rgb_in[1:, 5:].astype(np.float32) / np.float32(255.0))
                               .permute(0, 1, 4, 2, 3).contiguous(), DEV)
    assert np.array_equal(ref[1, 5:], fresh[0])             # the RGB stream restarted slot 1 from C[0]
    s = net.stream(2, h, w, device=DEV, input='nv12', out_format='nv12')
    got = np.concatenate([s.push(nv12[:, :3]), s.push(nv12[:, 3:5]), s.push(nv12[:, 5:], reset=[False, True])],
                         axis=1)
    want = Y.rgb_to_yuv420(ref, 'nv12')
    assert np.array_equal(got, want), int((got != want).sum())
    s.close()
    r.close()


def test_nv12_device_input_and_output(bd4_net):
    net = bd4_net
    c, h, w = BD4['c'], BD4['h'], BD4['w']
    nv12, _ = _yuv_clip(_clips_u8(53, 2, 6, c, h, w), 'nv12')
    want = _push_chunks(net.stream(2, h, w, device=DEV, input='nv12', out_format='nv12'), nv12, [3, 3])
    s = net.stream(2, h, w, device=DEV, input='nv12', out_format='nv12')
    dev_in = torch.from_numpy(nv12).to(DEV)
    o1 = s.push(dev_in[:, :3], out='device')           # a slice of the clip: frames contiguous, the chunk not
    H, W = 4 * h, 4 * w
    assert o1.is_cuda and o1.dtype == torch.uint8 and tuple(o1.shape) == (2, 3, 3 * H // 2, W)
    assert np.array_equal(o1.cpu().numpy(), want[:, :3])
    o1.fill_(0)                                       # the caller owns the result: the stream's buffers are separate
    o2 = s.push(dev_in[:, 3:], out='device')
    assert np.array_equal(o2.cpu().numpy(), want[:, 3:])
    assert int(o1.max()) == 0
    s.close()
