#!/usr/bin/env python
"""HR frames/s of streamed inference (FRNet.stream) against FRNet.infer_sequence on bench.py's bd4 workload:
4 lock-stepped clips of 3x134x320 LR (-> 3x536x1280), bench weights, --frames frames per clip.

    python tools/stream_bench.py [--frames 64] [--reps 3]

Prints one JSON line with, per path, the median and all --reps runs (HR frames/s = clips * frames / wall time;
each run ends in a device synchronisation; one untimed warm-up run of every path first):
  infer_sequence_fp32_host   FRNet.infer_sequence(pinned fp32 [n,t,c,h,w]) -> uint8 host
  push_u8_host_chunk1/16     VideoStream.push(pinned uint8 [n,k,h,w,c], out='host'), k = 1 / 16
  push_u8_device             VideoStream.push(uint8 on the device, out='device'), k = 16
  push_nv12_host_chunk1/16   VideoStream.push(pinned NV12 [n,k,3h/2,w], out='host') of an input='nv12',
                             out_format='nv12' stream -> NV12 [n,k,3H/2,W], k = 1 / 16
  push_nv12_device           the same with NV12 on the device and out='device', k = 16
  push_p010_709_host_chunk16 a P010 / BT.709 -> P010 / BT.709 stream (uint16 [n,k,3h/2,w] -> [n,k,3H/2,W]), k = 16
  push_nv12_601_709_host_chunk16  an NV12 / BT.601 -> NV12 / BT.709 stream, k = 16
  push_<yuy2|uyvy|i444>_host_chunk16  a YUY2 -> YUY2, UYVY -> UYVY or I444 -> I444 stream (BT.601 limited range;
                             uint8 [n,k,h,2w] / [n,k,3h,w] in and [n,k,H,2W] / [n,k,3H,W] out), k = 16
  frame_in_us                tg_stream_frame_in per step (decode of 4 frames, zero reset mask; and with every
                             slot reset) and tg_stream_frame_in_yuv420 per step (NV12, I420), CUDA events over a
                             graph of launches on rotating buffers
                             and tg_stream_frame_in_yuv per step (P010 / BT.709; YUY2, UYVY, I444 / BT.601;
                             I444_10 / BT.709), the last four with their algorithmic bytes (frames read, lr_curr
                             written) and TB/s in frame_in_422_444_tb_per_s
  push_u8_resize_<Ho>x<Wo>[_lanczos]_host_chunk16
                             an RGB stream with out_size=(Ho, Wo) (bicubic unless marked), k = 16: 402x960 (3/4) and
                             804x1920 (3/2)
  push_nv12_709_resize_402x960_host_chunk16  uint8 in, NV12 / BT.709 out at out_size=(402, 960), k = 16
  push_u8_scene_host_chunk1/16
                             push_u8_host_chunk1/16 on a stream with scene_cut=10 (the same frames have no cut, so
                             the bytes must equal infer_sequence's and no cut may be reported); each push's last_cuts
                             is read inside the timed pushes and summed over the timed reps (scene_cuts_reported);
                             alternates with the paths above in every rep
  resample_us                tg_resample_nchw_f32 per step (4 HR frames -> uint8 NHWC or fp32 NCHW), timed as below,
                             with its algorithmic bytes (n*3*H*W*4 read, n*Ho*Wo*3 or *12 written) and TB/s
  encode_us                  tg_rgb_u8_to_yuv420 per step (4 HR frames -> NV12 / I420) and tg_rgb_to_yuv per step
                             (uint8 -> NV12 / BT.709; fp32 NCHW -> P010 / BT.709; uint8 -> YUY2, UYVY, I444;
                             fp32 NCHW -> I444_10 / BT.709), timed the same way; the 4:2:2 / 4:4:4 ones with their
                             algorithmic bytes and TB/s in encode_422_444_tb_per_s
  scene_us                   tg_scene_cut per step (4 slots of 3x134x320 scored against another 4, with its
                             algorithmic bytes 2*n*c*h*w*4 and TB/s; 16 disjoint pairs of frame sets, 66 MB, rotate so
                             that L2 does not hold the next launch's input) and the reset-only tg_stream_frame_in that
                             follows it in the graph, on a step without cuts (an all-zero cut mask), timed the same way
All uint8 paths process the same frames (uint8, and the reference loader's float32 / 255 of them), so their
outputs are also compared byte for byte.  The NV12 paths take oracle/yuv_oracle.py's NV12 of those frames; their
output is compared with the oracle's NV12 of the RGB output for the frames that NV12 decodes to; the BT.709 NV12
output with oracle/yuv_color.py's BT.709 encode of that RGB output, and the P010 output with its encode of the fp32 HR
frames of a device loop of FRNet.step over the frames P010 decodes to.  The resized RGB outputs are compared with
oracle/resample.py's float64 resize of the fp32 HR frames of a device loop of FRNet.step (equal, or 1 apart where
x * 255 is within 1e-3 of a rounding boundary), the resized NV12 output with the BT.709 encode of the resized RGB
output.  The YUY2, UYVY and I444 outputs are compared with oracle/yuv_422_444.py's encode of the RGB output for the
frames each input decodes to.  Card name and power limit are read in the same run.  Writes nothing."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit_w():
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=20)
        return float(r.stdout.strip().splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=64)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if args.frames < 60:
        ap.error('--frames must be >= 60')
    import numpy as np
    import torch
    import bench
    import tecogan_b200 as T
    from oracle import yuv_oracle as Y
    from oracle import yuv_color as C
    from oracle import yuv_422_444 as C4
    from oracle import resample as R
    ops = sys.modules['tecogan-pytorch_b200.ops']
    assert torch.cuda.is_available(), 'stream_bench.py needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    bench.select_workload('bd4')
    n, (c, h, w), s = bench.CLIPS_PER_GPU, bench.LR, bench.SCALE
    t = args.frames
    net = T.FRNet(3, 3, 64, 10, 'BD', s)
    net.load_state_dict(bench.make_params(), strict=True)
    net = net.to(dev).eval()

    clips = bench.synthetic_clips(n, t, seed=100).numpy()                            # [n,t,c,h,w] in [0,1]
    u8 = np.ascontiguousarray(np.rint(clips * 255.0).astype(np.uint8).transpose(0, 1, 3, 4, 2))
    f32 = torch.from_numpy(u8.astype(np.float32) / np.float32(255.0)).permute(0, 1, 4, 2, 3).contiguous()
    f32_pin, u8_pin = f32.pin_memory(), torch.from_numpy(u8).pin_memory()
    u8_dev = u8_pin.to(dev)
    nv12 = Y.rgb_to_yuv420(u8, 'nv12')                                                # [n,t,3h/2,w]
    nv12_pin = torch.from_numpy(nv12).pin_memory()
    nv12_dev = nv12_pin.to(dev)
    p010 = C.rgb_to_yuv(np.rint(u8.astype(np.float64) * (1023.0 / 255.0)).astype(np.int64), 'p010', 'bt709')
    p010_pin = torch.from_numpy(p010).pin_memory()
    packed = {lay: C4.rgb_to_yuv(u8, lay) for lay in ('yuy2', 'uyvy', 'i444')}         # [n,t,h,2w] / [n,t,3h,w]
    packed_pin = {lay: torch.from_numpy(v).pin_memory() for lay, v in packed.items()}

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return n * t / (time.perf_counter() - t0), out

    def pushes(stream, src, chunk, out, cuts=None):
        res = []
        for i in range(0, t, chunk):
            res.append(stream.push(src[:, i:i + chunk], out=out))
            if cuts is not None:                 # a caller of a scene_cut stream reads each push's report
                cuts[0] += int(stream.last_cuts.sum())
        return res

    streams = {'push_u8_host_chunk1': (1, u8_pin, 'host'), 'push_u8_host_chunk16': (16, u8_pin, 'host'),
               'push_u8_device': (16, u8_dev, 'device'), 'push_nv12_host_chunk1': (1, nv12_pin, 'host'),
               'push_nv12_host_chunk16': (16, nv12_pin, 'host'), 'push_nv12_device': (16, nv12_dev, 'device'),
               'push_p010_709_host_chunk16': (16, p010_pin, 'host'),
               'push_nv12_601_709_host_chunk16': (16, nv12_pin, 'host')}
    kinds = {'push_p010_709_host_chunk16': dict(input='p010', out_format='p010', in_color='bt709', out_color='bt709'),
             'push_nv12_601_709_host_chunk16': dict(input='nv12', out_format='nv12', out_color='bt709')}
    resized = {'push_u8_resize_402x960_host_chunk16': dict(out_size=(402, 960)),
               'push_u8_resize_804x1920_host_chunk16': dict(out_size=(804, 1920)),
               'push_u8_resize_402x960_lanczos_host_chunk16': dict(out_size=(402, 960), resize_filter='lanczos'),
               'push_nv12_709_resize_402x960_host_chunk16': dict(out_size=(402, 960), out_format='nv12',
                                                                 out_color='bt709')}
    for k, kw in resized.items():
        streams[k] = (16, u8_pin, 'host')
        kinds[k] = kw
    for lay in packed:
        streams[f'push_{lay}_host_chunk16'] = (16, packed_pin[lay], 'host')
        kinds[f'push_{lay}_host_chunk16'] = dict(input=lay, out_format=lay)
    for chunk in (1, 16):
        streams[f'push_u8_scene_host_chunk{chunk}'] = (chunk, u8_pin, 'host')
        kinds[f'push_u8_scene_host_chunk{chunk}'] = dict(scene_cut=10.0)
    scene_cuts = {k: 0 for k in streams if 'scene' in k}
    opened = {k: net.stream(n, h, w, device=dev, **kinds.get(k, dict(input='nv12', out_format='nv12') if 'nv12' in k
                                                                 else {}))
              for k in streams}
    runs = {k: [] for k in ['infer_sequence_fp32_host', *streams]}
    outputs = {}
    # rep 0 is the untimed warm-up: graph capture, and the caching host allocator's pinned output blocks (each
    # path's previous output is dropped before its call, so later reps reuse them instead of pinning new memory)
    for rep in range(args.reps + 1):                                                 # paths alternate per rep
        outputs['infer_sequence_fp32_host'] = None
        fps, outputs['infer_sequence_fp32_host'] = timed(lambda: net.infer_sequence(f32_pin, dev))
        if rep:
            runs['infer_sequence_fp32_host'].append(fps)
        for k, (chunk, src, out) in streams.items():
            opened[k].reset(range(n))
            outputs[k] = None
            counter = [0] if k in scene_cuts else None
            fps, outputs[k] = timed(lambda: pushes(opened[k], src, chunk, out, counter))
            if rep:
                runs[k].append(fps)
                if counter is not None:
                    scene_cuts[k] += counter[0]
    ref = outputs['infer_sequence_fp32_host']
    # the NV12 paths' specification: the oracle's NV12 of the RGB output for the frames the NV12 input decodes to
    rgb_in = Y.yuv420_to_rgb(nv12, 'nv12')
    ref_rgb = net.infer_sequence(torch.from_numpy(rgb_in.astype(np.float32) / np.float32(255.0))
                                 .permute(0, 1, 4, 2, 3).contiguous(), dev)
    def p010_matches(got):
        """frame by frame against the oracle's P010 of the fp32 HR frames of a device loop of FRNet.step"""
        lr = torch.from_numpy((C.yuv_to_rgb(p010, 'p010', 'bt709').astype(np.float32) / np.float32(1023.0))
                              .transpose(0, 1, 4, 2, 3).copy())
        lr_prev = torch.zeros(n, c, h, w, device=dev)
        hr_prev = torch.zeros(n, c, s * h, s * w, device=dev)
        with torch.no_grad():
            for i in range(t):
                cur = lr[:, i].contiguous().to(dev)
                hr = net.step(cur, lr_prev, hr_prev)
                want = C.rgb_f32_to_yuv(hr.permute(0, 2, 3, 1).cpu().numpy(), 'p010', 'bt709')
                if not np.array_equal(got[:, i], want):
                    return False
                lr_prev, hr_prev = cur, hr
        return True

    hr_loop = None

    def resized_matches(got, size, filt):
        """frame by frame against the oracle's float64 resize of the fp32 HR frames of a device loop of FRNet.step
        (its dense matrices applied in float64 on the device), under the uint8 rule"""
        nonlocal hr_loop
        if hr_loop is None:
            hr_loop, lr_prev, hr_prev = [], torch.zeros(n, c, h, w, device=dev), torch.zeros(n, c, s * h, s * w,
                                                                                              device=dev)
            with torch.no_grad():
                for i in range(t):
                    cur = f32[:, i].to(dev)
                    hr_prev = net.step(cur, lr_prev, hr_prev)
                    lr_prev = cur
                    hr_loop.append(hr_prev.clone())
        my = torch.from_numpy(R.matrix(s * h, size[0], filt)).to(dev)
        mx = torch.from_numpy(R.matrix(s * w, size[1], filt)).to(dev)
        if got.shape != (n, t, *size, c):
            return False
        for i in range(t):            # R.to_uint8 and R.near_boundary, evaluated on the device
            ref = (my @ (hr_loop[i].double() @ mx.T)).permute(0, 2, 3, 1)
            q = torch.round(ref.float() * 255.0).clamp(0, 255).int()
            v = ref * 255.0
            near = (v - v.floor() - 0.5).abs() < 1e-3
            d = (torch.from_numpy(got[:, i]).to(dev).int() - q).abs()
            if int(d.max()) > 1 or bool((d[~near] > 0).any()):
                return False
        return True

    identical = {}
    for k, (chunk, src, out) in streams.items():
        got = np.concatenate([o.cpu().numpy() if out == 'device' else o for o in outputs[k]], axis=1)
        if k == 'push_nv12_709_resize_402x960_host_chunk16':
            rgb = np.concatenate(outputs['push_u8_resize_402x960_host_chunk16'], axis=1)
            identical[k] = got.shape == (n, t, 3 * 402 // 2, 960) and all(
                np.array_equal(got[j, i], C.rgb_to_yuv(rgb[j, i], 'nv12', 'bt709')) for j in range(n)
                for i in range(t))
        elif k in resized:
            identical[k] = resized_matches(got, resized[k]['out_size'], resized[k].get('resize_filter', 'bicubic'))
        elif k == 'push_p010_709_host_chunk16':
            identical[k] = got.shape == (n, t, 3 * s * h // 2, s * w) and p010_matches(got)
        elif k == 'push_nv12_601_709_host_chunk16':
            identical[k] = got.shape == (n, t, 3 * s * h // 2, s * w) and all(
                np.array_equal(got[j, i], C.rgb_to_yuv(ref_rgb[j, i], 'nv12', 'bt709')) for j in range(n)
                for i in range(t))
        elif k.startswith(tuple(f'push_{lay}_' for lay in packed)):
            lay = k.split('_')[1]
            rgb_lay = C4.yuv_to_rgb(packed[lay], lay)
            ref_lay = net.infer_sequence(torch.from_numpy(rgb_lay.astype(np.float32) / np.float32(255.0))
                                         .permute(0, 1, 4, 2, 3).contiguous(), dev)
            identical[k] = got.shape == (n, t, *C4.frame_shape(lay, s * h, s * w)) and all(
                np.array_equal(got[j, i], C4.rgb_to_yuv(ref_lay[j, i], lay)) for j in range(n) for i in range(t))
        elif 'nv12' in k:        # frame by frame: the oracle's int64 temporaries of a whole clip are GBs
            identical[k] = got.shape == (n, t, 3 * s * h // 2, s * w) and all(
                np.array_equal(got[j, i], Y.rgb_to_yuv420(ref_rgb[j, i], 'nv12')) for j in range(n) for i in range(t))
        else:
            identical[k] = bool(np.array_equal(got, ref))
    stream_launches = opened['push_u8_device']._engine.launches_per_step
    nv12_launches = opened['push_nv12_device']._engine.launches_per_step
    p010_launches = opened['push_p010_709_host_chunk16']._engine.launches_per_step
    resize_launches = opened['push_u8_resize_402x960_host_chunk16']._engine.launches_per_step
    scene_launches = opened['push_u8_scene_host_chunk16']._engine.launches_per_step
    for st in opened.values():
        st.close()

    # tg_stream_frame_in alone: 8 rotating buffer sets (8 x 4 x 2 MB of lr_curr), 60 launches per graph
    nb, reps = 8, 60
    H, W = s * h, s * w
    ins = [torch.randint(0, 256, (n, h, w, c), dtype=torch.uint8, device=dev) for _ in range(nb)]
    lrs = [torch.empty(n, c, h, w, device=dev) for _ in range(nb)]
    prev = torch.empty(n, c, h, w, device=dev)
    hrp = torch.empty(n, c, H, W, device=dev)
    frame_in = {}
    for name, val in (('decode', 0), ('decode_and_reset_all', 1)):
        mask = torch.full((n,), val, dtype=torch.int32, device=dev)
        sec = bench._time_graph(lambda i: ops.stream_frame_in(ins[i], mask, lrs[i], prev, hrp, s), nb, reps, torch)
        frame_in[name] = sec * 1e6
    yuv_ins = [torch.randint(0, 256, (n, 3 * h // 2, w), dtype=torch.uint8, device=dev) for _ in range(nb)]
    for layout in ('nv12', 'i420'):
        sec = bench._time_graph(lambda i: ops.stream_frame_in_yuv420(yuv_ins[i], layout, None, lrs[i], prev, hrp, s),
                                nb, reps, torch)
        frame_in[f'decode_{layout}'] = sec * 1e6
    p010_ins = [torch.randint(0, 1 << 15, (n, 3 * h // 2, w), dtype=torch.int16, device=dev).view(torch.uint16)
                for _ in range(nb)]
    sec = bench._time_graph(lambda i: ops.stream_frame_in_yuv(p010_ins[i], 'p010', 'bt709', None, lrs[i], prev, hrp, s),
                            nb, reps, torch)
    frame_in['decode_p010_bt709'] = sec * 1e6
    frame_in_bytes = {}
    for lay, color in (('yuy2', 'bt601'), ('uyvy', 'bt601'), ('i444', 'bt601'), ('i444_10', 'bt709')):
        shape = (n, *C4.frame_shape(lay, h, w))
        src = [torch.randint(0, 1 << 15, shape, dtype=torch.int16, device=dev).view(torch.uint16) if lay == 'i444_10'
               else torch.randint(0, 256, shape, dtype=torch.uint8, device=dev) for _ in range(nb)]
        sec = bench._time_graph(lambda i: ops.stream_frame_in_yuv(src[i], lay, color, None, lrs[i], prev, hrp, s),
                                nb, reps, torch)
        frame_in[f'decode_{lay}_{color}'] = sec * 1e6
        frame_in_bytes[f'decode_{lay}_{color}'] = src[0].numel() * src[0].element_size() + n * c * h * w * 4
        del src
    # tg_rgb_u8_to_yuv420 alone: 8 rotating sets of 4 HR frames (8 x 8.2 MB in, 8 x 4.1 MB out)
    rgbs = [torch.randint(0, 256, (n, H, W, c), dtype=torch.uint8, device=dev) for _ in range(nb)]
    yuvs = [torch.empty(n, 3 * H // 2, W, dtype=torch.uint8, device=dev) for _ in range(nb)]
    encode = {}
    for layout in ('nv12', 'i420'):
        sec = bench._time_graph(lambda i: ops.rgb_u8_to_yuv420(rgbs[i], layout, out=yuvs[i]), nb, reps, torch)
        encode[layout] = sec * 1e6
    sec = bench._time_graph(lambda i: ops.rgb_to_yuv('nv12', 'bt709', rgb_u8=rgbs[i], out=yuvs[i]), nb, reps, torch)
    encode['nv12_bt709'] = sec * 1e6
    hrs = [torch.rand(n, c, H, W, device=dev) for _ in range(nb)]
    p010s = [torch.empty(n, 3 * H // 2, W, dtype=torch.uint16, device=dev) for _ in range(nb)]
    sec = bench._time_graph(lambda i: ops.rgb_to_yuv('p010', 'bt709', rgb_f32=hrs[i], out=p010s[i]), nb, reps, torch)
    encode['p010_bt709'] = sec * 1e6
    encode_new_bytes = {}
    for lay in ('yuy2', 'uyvy', 'i444'):
        outs = [torch.empty(n, *C4.frame_shape(lay, H, W), dtype=torch.uint8, device=dev) for _ in range(nb)]
        sec = bench._time_graph(lambda i: ops.rgb_to_yuv(lay, 'bt601', rgb_u8=rgbs[i], out=outs[i]), nb, reps, torch)
        encode[lay] = sec * 1e6
        encode_new_bytes[lay] = n * H * W * 3 + outs[0].numel()
        del outs
    outs = [torch.empty(n, 3 * H, W, dtype=torch.uint16, device=dev) for _ in range(nb)]
    sec = bench._time_graph(lambda i: ops.rgb_to_yuv('i444_10', 'bt709', rgb_f32=hrs[i], out=outs[i]), nb, reps,
                            torch)
    encode['i444_10_bt709'] = sec * 1e6
    encode_new_bytes['i444_10_bt709'] = n * c * H * W * 4 + n * 3 * H * W * 2
    del outs
    encode_bytes = n * H * W * 3 + n * 3 * H // 2 * W
    # tg_resample_nchw_f32 alone: the same 8 rotating sets of 4 fp32 HR frames (8 x 33 MB)
    resample, resample_bytes = {}, {}
    for name, (Ho, Wo), filt, f32_out in (('u8_402x960_bicubic', (402, 960), 'bicubic', False),
                                          ('u8_804x1920_bicubic', (804, 1920), 'bicubic', False),
                                          ('u8_402x960_lanczos', (402, 960), 'lanczos', False),
                                          ('f32_402x960_bicubic', (402, 960), 'bicubic', True)):
        tabs = [tuple(v.to(dev) for v in ops.resample_table(a, b, filt)) for a, b in ((H, Ho), (W, Wo))]
        outs = [torch.empty((n, c, Ho, Wo) if f32_out else (n, Ho, Wo, c), dtype=torch.float32 if f32_out else
                            torch.uint8, device=dev) for _ in range(nb)]
        kw = (lambda i: {'out_f32': outs[i]}) if f32_out else (lambda i: {'out_u8': outs[i]})
        sec = bench._time_graph(lambda i: ops.resample(hrs[i], *tabs, **kw(i)), nb, reps, torch)
        resample[name] = sec * 1e6
        resample_bytes[name] = n * c * H * W * 4 + n * Ho * Wo * c * (4 if f32_out else 1)
        del outs
    encode10_bytes = n * H * W * 3 * 4 + n * 3 * H // 2 * W * 2
    # tg_scene_cut alone: 16 disjoint (current, previous) pairs of 4 x 3x134x320 fp32 frames (66 MB, more than the
    # 50 MB L2), then the reset-only tg_stream_frame_in with an all-zero cut mask (what the graph runs on a step
    # without cuts)
    ns = 16
    scene_a = [torch.rand(n, c, h, w, device=dev) for _ in range(ns)]
    scene_b = [torch.rand(n, c, h, w, device=dev) for _ in range(ns)]
    prev_mafd = torch.full((n,), -1.0, dtype=torch.float64, device=dev)
    work = ops.scene_cut_work(n, dev)
    score = torch.empty(n, dtype=torch.float64, device=dev)
    cut = torch.zeros(n, dtype=torch.int32, device=dev)
    no_reset = torch.zeros(n, dtype=torch.int32, device=dev)
    scene = {}
    sec = bench._time_graph(lambda i: ops.scene_cut(scene_a[i], scene_b[i], no_reset, 10.0, prev_mafd, work, score,
                                                    cut), ns, reps, torch)
    scene['scene_cut'] = sec * 1e6
    del scene_a, scene_b
    cut.zero_()                          # the scene_cut launches above left their own flags in cut
    sec = bench._time_graph(lambda i: ops.stream_frame_in(None, cut, lrs[i], prev, hrp, s), nb, reps, torch)
    scene['reset_only_frame_in_no_cut'] = sec * 1e6
    scene_bytes = 2 * n * c * h * w * 4

    line = {
        'metric': 'hr_frames_per_sec_4xBD_3x134x320_streamed', 'unit': 'frames/s',
        'device': torch.cuda.get_device_name(0), 'power_limit_w': power_limit_w(),
        'clips': n, 'frames_per_clip': t, 'reps': args.reps,
        'results': {k: {'median': statistics.median(v), 'runs': v} for k, v in runs.items()},
        'identical_to_infer_sequence': identical,
        'frame_in_us': frame_in,
        'encode_us': encode,
        'resample_us': resample,
        'scene_us': scene,
        'scene_bytes_per_step': scene_bytes,
        'scene_tb_per_s': scene_bytes / scene['scene_cut'] * 1e-6,
        'scene_cuts_reported': scene_cuts,          # summed over the timed pushes of every timed rep
        'resample_bytes_per_step': resample_bytes,
        'resample_tb_per_s': {k: resample_bytes[k] / v * 1e-6 for k, v in resample.items()},
        'encode_bytes_per_step': encode_bytes,
        'encode10_bytes_per_step': encode10_bytes,
        'encode_gb_per_s': {k: (encode10_bytes if k.startswith('p010') else encode_bytes) / v * 1e-3
                            for k, v in encode.items() if k not in encode_new_bytes},
        'frame_in_422_444_bytes_per_step': frame_in_bytes,
        'frame_in_422_444_tb_per_s': {k: b / frame_in[k] * 1e-6 for k, b in frame_in_bytes.items()},
        'encode_422_444_bytes_per_step': encode_new_bytes,
        'encode_422_444_tb_per_s': {k: b / encode[k] * 1e-6 for k, b in encode_new_bytes.items()},
        'h2d_bytes_per_step': {'fp32': n * c * h * w * 4, 'uint8': n * c * h * w, 'nv12': n * 3 * h // 2 * w},
        'd2h_bytes_per_step': {'uint8': n * c * H * W, 'nv12': n * 3 * H // 2 * W},
        'launches_per_step': {'infer_sequence': T.engine.get_engine(net, n, c, h, w, dev).launches_per_step,
                              'push': stream_launches, 'push_nv12': nv12_launches, 'push_p010': p010_launches,
                              'push_resize': resize_launches, 'push_scene': scene_launches},
    }
    print(json.dumps(line), flush=True)


if __name__ == '__main__':
    main()
