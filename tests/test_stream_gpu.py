"""pytest -m gpu: streamed inference (FRNet.stream / VideoStream.push) and its frame-input kernel
tg_stream_frame_in.

- the kernel converts uint8 to float32 / 255 bit for bit as the reference's loader does (numpy float32 division),
  in RGB and BGR order, at ragged widths and from misaligned sources, and its reset zeroes only flagged slots;
- pushing a clip in chunks gives the bytes of one infer_sequence call on the whole clip (4x BD at the bench
  shape and weights, and 2x BI at a small shape), for uint8 and fp32 input;
- a slot reset in the middle of a stream restarts that slot exactly and leaves the other slot untouched;
- device input and output give the host path's bytes and never alias the engine's buffers."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
BD4 = dict(scale=4, degradation='BD', c=3, h=134, w=320)      # bench.py's bd4 frame
BI2 = dict(scale=2, degradation='BI', c=3, h=36, w=52)


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


def _to_f32(u8):
    """The reference loader's conversion (paired_folder_dataset.py:49) in numpy: [n,t,h,w,c] -> torch [n,t,c,h,w]."""
    return torch.from_numpy(np.ascontiguousarray((u8.astype(np.float32) / np.float32(255.0)).transpose(0, 1, 4, 2, 3)))


def _push_chunks(stream, frames, chunks, **kw):
    out, i = [], 0
    for k in chunks:
        out.append(stream.push(frames[:, i:i + k], **kw))
        i += k
    assert i == frames.shape[1]
    return np.concatenate(out, axis=1)


# ------------------------------------------------------------------------------------------------ kernel
def _frame_in(u8, reset, lr_curr, lr_prev, hr_prev, scale, bgr):
    ops.stream_frame_in(u8, reset, lr_curr, lr_prev, hr_prev, scale, bgr=bgr)
    torch.cuda.synchronize()


@pytest.mark.parametrize('bgr', [False, True], ids=['rgb', 'bgr'])
@pytest.mark.parametrize('n,h,w,offset', [(1, 16, 16, 0), (3, 37, 53, 0), (3, 37, 53, 5), (2, 7, 5, 13)])
def test_frame_in_decodes_bit_exactly(n, h, w, offset, bgr):
    """Every uint8 value (the 16x16 frame holds 0..255 three times) and random frames whose rows are not a multiple
    of 16 bytes, read from a source `offset` bytes past a 16-byte boundary."""
    c, s = 3, 4
    rng = np.random.default_rng(100 + n + h + offset)
    if h == 16:
        img = np.arange(n * h * w * c, dtype=np.int64).reshape(n, h, w, c) % 256
        img = img.astype(np.uint8)
    else:
        img = rng.integers(0, 256, size=(n, h, w, c), dtype=np.uint8)
    buf = torch.zeros(offset + img.size + 16, dtype=torch.uint8, device=DEV)
    u8 = buf[offset:offset + img.size].view(n, h, w, c)
    u8.copy_(torch.from_numpy(img))
    lr = torch.full((n, c, h, w), float('nan'), device=DEV)
    prev = torch.full_like(lr, 3.0)
    hr = torch.full((n, c, s * h, s * w), 5.0, device=DEV)
    _frame_in(u8, None, lr, prev, hr, s, bgr)
    src = img[..., ::-1] if bgr else img
    want = src.astype(np.float32).transpose(0, 3, 1, 2) / np.float32(255.0)
    got = lr.cpu().numpy()
    assert got.dtype == np.float32 and np.array_equal(got.view(np.uint32), want.view(np.uint32))
    assert bool((prev == 3.0).all()) and bool((hr == 5.0).all())          # no reset mask: state untouched


@pytest.mark.parametrize('with_frames', [True, False], ids=['decode_and_reset', 'reset_only'])
def test_frame_in_reset_zeroes_flagged_slots_only(with_frames):
    n, c, h, w, s = 3, 3, 37, 53, 4         # a slot of lr_prev is 5883 floats: its start is not 16-byte aligned
    g = torch.Generator(device=DEV).manual_seed(7)
    lr = torch.full((n, c, h, w), float('nan'), device=DEV)
    prev = torch.rand((n, c, h, w), generator=g, device=DEV) + 1.0
    hr = torch.rand((n, c, s * h, s * w), generator=g, device=DEV) + 1.0
    prev0, hr0 = prev.clone(), hr.clone()
    u8 = torch.randint(0, 256, (n, h, w, c), generator=g, device=DEV, dtype=torch.uint8) if with_frames else None
    mask = torch.tensor([1, 0, 1], dtype=torch.int32, device=DEV)
    _frame_in(u8, mask, lr, prev, hr, s, False)
    for k in (0, 2):
        assert bool((prev[k] == 0).all()) and bool((hr[k] == 0).all()), k
    assert torch.equal(prev[1].view(torch.int32), prev0[1].view(torch.int32))
    assert torch.equal(hr[1].view(torch.int32), hr0[1].view(torch.int32))
    if with_frames:
        want = u8.permute(0, 3, 1, 2).cpu().numpy().astype(np.float32) / np.float32(255.0)
        assert np.array_equal(lr.cpu().numpy(), want)
    else:
        assert bool(torch.isnan(lr).all())                                  # in_u8 = NULL: lr_curr is not written
    mask.zero_()
    _frame_in(u8, mask, lr, prev0, hr0, s, False)                          # an all-zero mask writes nothing
    assert bool((prev0 > 0).all()) and bool((hr0 > 0).all())


# ------------------------------------------------------------------------------------------------ streams
@pytest.mark.parametrize('geom', [BD4, BI2], ids=['bd4', 'bi2'])
def test_chunked_push_matches_infer_sequence(geom, bd4_net):
    """n=2 clips of 10 frames pushed as chunks [1,4,2,3]: uint8 input, fp32 input and BGR uint8 input all give the
    bytes of one infer_sequence call on the reference loader's fp32 frames."""
    net = bd4_net if geom is BD4 else _net(geom['scale'], geom['degradation'])
    c, h, w = geom['c'], geom['h'], geom['w']
    u8 = _clips_u8(11, 2, 10, c, h, w)
    f32 = _to_f32(u8)
    ref = net.infer_sequence(f32.pin_memory(), DEV)                        # [n,t,H,W,c]
    chunks = [1, 4, 2, 3]
    got = _push_chunks(net.stream(2, h, w, device=DEV), torch.from_numpy(u8), chunks)
    assert got.shape == ref.shape and got.dtype == np.uint8
    assert np.array_equal(got, ref), int((got != ref).sum())
    got = _push_chunks(net.stream(2, h, w, device=DEV, input='float32'), f32, chunks)
    assert np.array_equal(got, ref), int((got != ref).sum())
    bgr = np.ascontiguousarray(u8[..., ::-1])
    got = _push_chunks(net.stream(2, h, w, device=DEV, channel_order='bgr'), bgr, chunks)   # NumPy input
    assert np.array_equal(got, ref), int((got != ref).sum())


def test_slot_reset_restarts_one_slot(bd4_net):
    """Slot 1 switches from video B to video C at frame 5 while slot 0 plays video A throughout."""
    net = bd4_net
    c, h, w = BD4['c'], BD4['h'], BD4['w']
    a, b, cc = (_clips_u8(seed, 1, 10, c, h, w) for seed in (21, 31, 41))
    frames = np.concatenate([a, np.concatenate([b[:, :5], cc[:, :5]], axis=1)], axis=0)    # [2,10,h,w,c]
    s = net.stream(2, h, w, device=DEV)
    parts = [s.push(frames[:, :3]), s.push(frames[:, 3:5]), s.push(frames[:, 5:], reset=[False, True])]
    got = np.concatenate(parts, axis=1)
    no_reset = net.infer_sequence(_to_f32(frames), DEV)
    assert np.array_equal(got[0], no_reset[0]), int((got[0] != no_reset[0]).sum())
    assert np.array_equal(got[1, :5], no_reset[1, :5])
    fresh = net.infer_sequence(_to_f32(np.concatenate([a[:, 5:], cc[:, :5]], axis=0)), DEV)   # slot 1 from C[0]
    assert np.array_equal(got[1, 5:], fresh[1]), int((got[1, 5:] != fresh[1]).sum())
    # the same restart requested through VideoStream.reset before the push
    s2 = net.stream(2, h, w, device=DEV)
    s2.push(frames[:, :5])
    s2.reset([1])
    assert np.array_equal(s2.push(frames[:, 5:]), got[:, 5:])
    s.close()
    s2.close()


def test_device_input_and_output(bd4_net):
    net = bd4_net
    c, h, w = BD4['c'], BD4['h'], BD4['w']
    u8 = _clips_u8(51, 2, 6, c, h, w)
    want = _push_chunks(net.stream(2, h, w, device=DEV), torch.from_numpy(u8), [3, 3])
    s = net.stream(2, h, w, device=DEV)
    dev_u8 = torch.from_numpy(u8).to(DEV)
    o1 = s.push(dev_u8[:, :3], out='device')          # a slice of the clip: frames contiguous, the chunk not
    assert o1.is_cuda and o1.dtype == torch.uint8 and tuple(o1.shape) == (2, 3, 4 * h, 4 * w, c)
    assert np.array_equal(o1.cpu().numpy(), want[:, :3])
    o1.fill_(0)                                      # the caller owns the result: the stream's buffers are separate
    o2 = s.push(dev_u8[:, 3:], out='device')
    assert np.array_equal(o2.cpu().numpy(), want[:, 3:])
    assert int(o1.max()) == 0
