"""pytest -m gpu: streamed inference with a resized output, FRNet.stream(out_size=, resize_filter=), end to end at
bench.py's bd4 shape and a small 2x BI shape.

The specification of every resized frame is oracle/resample.py's float64 resize of the fp32 HR frames of a device
loop of FRNet.step over the same frames, then the output's quantisation: uint8 as float32_to_uint8 (a difference
of 1 only where x * 255 lies within 1e-3 of a rounding boundary), NV12 as oracle/yuv_color.py's encode of that uint8
frame, P010 as its 10-bit encode of the fp32 resize."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import resample as R              # noqa: E402
from oracle import yuv_color as C              # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
BD4 = dict(scale=4, degradation='BD', c=3, h=134, w=320, out=(402, 960), filt='bicubic')    # 536x1280 -> 3/4
BI2 = dict(scale=2, degradation='BI', c=3, h=36, w=52, out=(54, 130), filt='lanczos')       # 72x104 -> 3/4 x 5/4
CHUNKS, RESETS, RESET_AT = [1, 4, 2, 3], [None, None, [False, True], None], {(1, 5)}


def _net(scale, degradation):
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def bd4_net():
    return _net(4, 'BD')


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


def _hr_loop(net, u8, resets):
    """fp32 HR frames [n,t,3,H,W] (device) of a device loop of net.step over u8 / 255, zero state at frame 0 and for
    slot k at frame i when (k, i) in resets.  The division is numpy's IEEE float32 one, the stream's decode (torch's
    CUDA division by a scalar multiplies by the reciprocal, which differs in the last bit)."""
    n, t = u8.shape[:2]
    lr = torch.from_numpy(np.ascontiguousarray((u8.astype(np.float32) / np.float32(255.0)).transpose(0, 1, 4, 2, 3)))
    lr = lr.to(DEV)
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


def _oracle_resize(hr, out_hw, filt):
    """oracle/resample.py's float64 resize of device fp32 frames [..., H, W] -> numpy float64 [..., Ho, Wo]: its
    dense per-axis matrices, applied in float64 on the device."""
    H, W = hr.shape[-2:]
    my = torch.from_numpy(R.matrix(H, out_hw[0], filt)).to(DEV)
    mx = torch.from_numpy(R.matrix(W, out_hw[1], filt)).to(DEV)
    return (my @ (hr.double() @ mx.T)).cpu().numpy()


def _check_u8(got, ref):
    """got uint8 [..., Ho, Wo, 3] against float64 ref [..., 3, Ho, Wo] under the uint8 rule.  The kernel's fp32 sums
    are within a few float32 ulps of the largest magnitude they add, so the rounding-boundary window (1e-3 of a code
    value for frames in [0, 1], as in the kernel tests) widens with the HR frames' range."""
    tol = 1e-3 * max(1.0, float(np.abs(ref).max()))
    ref = np.moveaxis(ref, -3, -1)
    diff = np.abs(got.astype(np.int32) - R.to_uint8(ref).astype(np.int32))
    near = R.near_boundary(ref, tol)
    assert diff.max() <= 1 and not (diff[~near] > 0).any(), (int((diff > 0).sum()), int(near.sum()))


def _geom(geom, bd4_net):
    net = bd4_net if geom is BD4 else _net(geom['scale'], geom['degradation'])
    return net, geom['c'], geom['h'], geom['w'], geom['out'], geom['filt']


@pytest.mark.parametrize('geom', [BD4, BI2], ids=['bd4', 'bi2'])
def test_resized_rgb_nv12_p010_match_oracle(geom, bd4_net):
    """n=2 clips of 10 frames pushed as [1,4,2,3] with slot 1 restarting at frame 5, host and device output."""
    net, c, h, w, size, filt = _geom(geom, bd4_net)
    u8 = _clips_u8(71, 2, 10, c, h, w)
    hr = _hr_loop(net, u8, RESET_AT)                                   # [n,t,3,H,W] on the device
    ref = _oracle_resize(hr, size, filt)                               # [n,t,3,Ho,Wo] float64
    tabs = [tuple(t.to(DEV) for t in ops.resample_table(a, b, filt)) for a, b in zip(hr.shape[-2:], size)]
    frames = [hr[:, i].contiguous() for i in range(hr.shape[1])]
    # the kernel alone on the loop's HR frames: the stream's outputs are these, byte for byte
    rgb_k = np.stack([ops.resample(x, *tabs).cpu().numpy() for x in frames], axis=1)
    f32 = torch.stack([ops.resample(x, *tabs, out_f32=torch.empty(2, 3, *size, device=DEV)) for x in frames],
                      dim=1).permute(0, 1, 3, 4, 2).cpu().numpy()
    _check_u8(rgb_k, ref)
    for out in ('host', 'device'):
        s = net.stream(2, h, w, device=DEV, out_size=size, resize_filter=filt)
        rgb = _push(s, u8, CHUNKS, RESETS, out)
        s.close()
        assert rgb.shape == (2, 10, *size, 3) and rgb.dtype == np.uint8
        assert np.array_equal(rgb, rgb_k), (out, int((rgb != rgb_k).sum()))
        # NV12 / BT.709: the 8-bit encode of that uint8 frame
        s = net.stream(2, h, w, device=DEV, out_format='nv12', out_color='bt709', out_size=size, resize_filter=filt)
        got = _push(s, u8, CHUNKS, RESETS, out)
        s.close()
        assert np.array_equal(got, C.rgb_to_yuv(rgb, 'nv12', 'bt709')), out
        # P010 / BT.709: the 10-bit encode of the kernel's fp32 resize of the loop's HR frames, exactly, and of the
        # oracle's float64 resize within 1 code value
        s = net.stream(2, h, w, device=DEV, out_format='p010', out_color='bt709', out_size=size, resize_filter=filt)
        got = _push(s, u8, CHUNKS, RESETS, out)
        s.close()
        assert np.array_equal(got, C.rgb_f32_to_yuv(f32, 'p010', 'bt709')), out
        want = C.rgb_f32_to_yuv(np.moveaxis(ref, -3, -1).astype(np.float32), 'p010', 'bt709')
        d = np.abs((got >> 6).astype(np.int32) - (want >> 6).astype(np.int32))
        assert d.max() <= 1 and (d > 0).mean() < 1e-2, (int(d.max()), float((d > 0).mean()))


@pytest.mark.parametrize('geom', [BD4, BI2], ids=['bd4', 'bi2'])
def test_chunks_resets_and_identity_size(geom, bd4_net):
    net, c, h, w, size, filt = _geom(geom, bd4_net)
    u8 = _clips_u8(83, 2, 10, c, h, w)
    for fmt in ('rgb', 'nv12', 'p010'):
        kw = dict(out_format=fmt, out_color='bt709' if fmt != 'rgb' else 'bt601')
        one = _push(net.stream(2, h, w, device=DEV, out_size=size, resize_filter=filt, **kw), u8, [10])
        chunked = _push(net.stream(2, h, w, device=DEV, out_size=size, resize_filter=filt, **kw), u8, CHUNKS)
        assert np.array_equal(one, chunked), fmt
        # a reset of slot 1 at frame 5 leaves slot 0 byte-identical
        reset = _push(net.stream(2, h, w, device=DEV, out_size=size, resize_filter=filt, **kw), u8, CHUNKS, RESETS)
        assert np.array_equal(reset[0], one[0]) and np.array_equal(reset[1, :5], one[1, :5]), fmt
        assert not np.array_equal(reset[1, 5:], one[1, 5:]), fmt
        # out_size = (H, W): the bytes of the stream without it
        H, W = net.scale * h, net.scale * w
        for f in ('bicubic', 'lanczos'):
            same = _push(net.stream(2, h, w, device=DEV, out_size=(H, W), resize_filter=f, **kw), u8, CHUNKS, RESETS)
            plain = _push(net.stream(2, h, w, device=DEV, **kw), u8, CHUNKS, RESETS)
            assert np.array_equal(same, plain), (fmt, f)


def test_resize_launches_per_step(bd4_net):
    """The resize is one launch per step.  The step drops its uint8 output when resizing: with the fused tail that
    output is free (written by the tail kernel), so the resized stream has one launch more; with the other tails
    (the default 'acc' one too) it is a launch of its own, which the resize replaces."""
    extra = 1 if ops.tail_mode() == 'fused' else 0
    u8 = _clips_u8(5, 4, 1, 3, 134, 320)
    for fmt in ('rgb', 'nv12', 'p010'):
        kw = dict(out_format=fmt)
        plain = bd4_net.stream(4, 134, 320, device=DEV, **kw)
        plain.push(u8)
        resized = bd4_net.stream(4, 134, 320, device=DEV, out_size=(402, 960), **kw)
        resized.push(u8)
        assert resized._engine.launches_per_step == plain._engine.launches_per_step + extra, fmt
        plain.close()
        resized.close()
