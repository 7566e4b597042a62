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
frames each input decodes to.  Card name and power limit are read in the same run.  Writes nothing.

    python tools/stream_bench.py --yuv422-10 [--frames 64] [--reps 3]

measures 10-bit 4:2:2 video instead (one JSON line, metric hr_frames_per_sec_4xBD_3x134x320_streamed_yuv422_10):
VideoStream.push of pinned frames, k = 16, out='host', in and out of one format -- rgb (uint8), p010_709, p210_709,
i422_10_709 and v210_709 (BT.709 limited range) -- the arms alternating in every rep, with the median, min, max and
runs of each; identical: P210's output frame by frame against oracle/yuv_422_10.py's encode of the fp32 HR frames of a
device loop of FRNet.step over its decode, I422_10's and v210's samples against P210's.  decode_us / encode_us:
tg_stream_frame_in_yuv and tg_rgb_to_yuv (from the fp32 HR frame) per step for P010 and the three layouts, CUDA events
over a graph of launches on 8 rotating buffer sets, with their algorithmic bytes (frames read or written, lr_curr or
the fp32 HR frame) and TB/s.  The card, its power limit and SM clocks (current, max) are read in the same run.

    python tools/stream_bench.py --window [--frames 64] [--reps 3]

measures letterboxed video instead (one JSON line, metric hr_frames_per_sec_4xBD_letterbox_134x320_in_180x320): the
bd4 clips as a 2.39:1 134x320 picture at row 22 of black 180x320 (16:9) frames, uint8 RGB -> RGB and NV12 -> NV12,
k = 16 pushes of pinned frames, three arms alternating in every rep:
  uncropped       today's path: the whole 180x320 frame through the net (-> 720x1280)
  crop_out_frame  crop=(22, 0, 134, 320), out_frame=(720, 1280): the picture through the net, placed in black
  precropped      a plain 134x320 stream over frames cropped on the host (-> 536x1280)
with crop_out_frame's output checked against precropped's placed into the black frame (oracle/frame_window.py), and
the kernel times of the windowed frame input and output writers next to the plain ones (CUDA events over graphs).

    python tools/stream_bench.py --pad [--frames 64] [--reps 3]

measures temporally padded streams instead (one JSON line, metric hr_frames_per_sec_4xBD_pad5): the bd4 clips, uint8
RGB -> RGB, k = 16 pushes of pinned frames and a flush, four arms alternating in every rep:
  plain / pad5            pad_front=0 and pad_front=5 reflect, clips without cuts
  plain_cuts32 / pad5_cuts32  the same with scene_cut=10 on clips that change shot every 32 frames in every slot
(reported cuts counted, so the cut arms must find n * (frames / 32 - 1) of them), then with CUDA events: one batch-n
warm-up step of the padded stream and one of a batch-1 padded stream (the cost of a warm start is p such steps), and
tg_stream_gather per step with all slots kept (the current frame copied) and all slots loaded, with its bytes.

    python tools/stream_bench.py --insize [--frames 64] [--reps 3]

measures a resized input instead (one JSON line, metric hr_frames_per_sec_4xBD_nv12_1080p_insize_540x960): the bd4
net (10 blocks, bench weights) on 1920x1080 NV12 sources with in_size=(540, 960), NV12 2160x3840 out, against the
same stream fed 960x540 NV12 frames directly, at n = 1 and n = 2 slots; k = 16 pushes of pinned frames (16 distinct
frames per slot, pushed again for every chunk) with out='device', the four arms alternating in every rep.  Then, in a
separate torch.profiler run of 16 frames of each stream, the frame-input kernel's time per step with its algorithmic
bytes (the NV12 frames read, lr_curr written) and TB/s.  The launch count per step of both streams is reported; it
must be the same."""
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
    ap.add_argument('--window', action='store_true', help='the letterboxed-video arms instead')
    ap.add_argument('--pad', action='store_true', help='the temporally padded arms instead')
    ap.add_argument('--insize', action='store_true', help='the resized-input arms instead')
    ap.add_argument('--yuv422-10', action='store_true', help='the 10-bit 4:2:2 (P210, I422_10, v210) arms instead')
    args = ap.parse_args()
    if args.frames < 60:
        ap.error('--frames must be >= 60')
    if args.window:
        return window_bench(args)
    if args.pad:
        return pad_bench(args)
    if args.insize:
        return insize_bench(args)
    if args.yuv422_10:
        return yuv422_10_bench(args)
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


def window_bench(args):
    import numpy as np
    import torch
    import bench
    import tecogan_b200 as T
    from oracle import frame_window as FW
    from oracle import yuv_oracle as Y
    ops = sys.modules['tecogan-pytorch_b200.ops']
    assert torch.cuda.is_available(), 'stream_bench.py needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    bench.select_workload('bd4')
    n, (c, h, w), s = bench.CLIPS_PER_GPU, bench.LR, bench.SCALE
    t, chunk = args.frames, 16
    Hf, top = 180, 22                      # 134 x 320 (2.39:1) at row 22 of 180 x 320 (16:9)
    box = (top, 0, h, w)
    net = T.FRNet(3, 3, 64, 10, 'BD', s)
    net.load_state_dict(bench.make_params(), strict=True)
    net = net.to(dev).eval()
    clips = bench.synthetic_clips(n, t, seed=100).numpy()
    pic = np.ascontiguousarray(np.rint(clips * 255.0).astype(np.uint8).transpose(0, 1, 3, 4, 2))   # [n,t,h,w,c]
    full = np.zeros((n, t, Hf, w, c), np.uint8)
    full[:, :, top:top + h] = pic
    src = {'uint8': (full, pic), 'nv12': (Y.rgb_to_yuv420(full, 'nv12'), None)}
    src['nv12'] = (src['nv12'][0], np.stack([np.stack([FW.crop_words(f, 'nv12', *box) for f in clip])
                                             for clip in src['nv12'][0]]))
    arms, opened, runs, outputs = {}, {}, {}, {}
    for fmt, (whole, cropped) in src.items():
        kw = dict(input=fmt, out_format='rgb' if fmt == 'uint8' else 'nv12')
        pins = torch.from_numpy(whole).pin_memory(), torch.from_numpy(np.ascontiguousarray(cropped)).pin_memory()
        arms[f'{fmt}_uncropped'] = (net.stream(n, Hf, w, device=dev, **kw), pins[0])
        arms[f'{fmt}_crop_out_frame'] = (net.stream(n, Hf, w, device=dev, crop=box, out_frame=(s * Hf, s * w), **kw),
                                         pins[0])
        arms[f'{fmt}_precropped'] = (net.stream(n, h, w, device=dev, **kw), pins[1])
    for k in arms:
        runs[k] = []
    for rep in range(args.reps + 1):                 # rep 0: untimed warm-up (graph capture, pinned blocks)
        for k, (st, frames) in arms.items():
            st.reset(range(n))
            outputs[k] = None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outputs[k] = [st.push(frames[:, i:i + chunk]) for i in range(0, t, chunk)]
            torch.cuda.synchronize()
            if rep:
                runs[k].append(n * t / (time.perf_counter() - t0))
    identical = {}
    for fmt in src:
        got = np.concatenate(outputs[f'{fmt}_crop_out_frame'], 1)
        ref = np.concatenate(outputs[f'{fmt}_precropped'], 1)
        lay = 'rgb' if fmt == 'uint8' else 'nv12'
        y, x = arms[f'{fmt}_crop_out_frame'][0].out_origin
        identical[fmt] = all(np.array_equal(got[j, i], FW.place_words(ref[j, i], lay, 'bt601', s * Hf, s * w, y, x))
                             for j in range(n) for i in range(t))
    launches = {k: st._engine.launches_per_step for k, (st, _) in arms.items()}
    for st, _ in arms.values():
        st.close()

    # the windowed kernels next to the plain ones: 8 rotating buffer sets, 60 launches per graph
    nb, reps = 8, 60
    H, W = s * h, s * w
    lrs = [torch.empty(n, c, h, w, device=dev) for _ in range(nb)]
    prev, hrp = torch.empty(n, c, h, w, device=dev), torch.empty(n, c, H, W, device=dev)
    rgb_full = [torch.randint(0, 256, (n, Hf, w, c), dtype=torch.uint8, device=dev) for _ in range(nb)]
    rgb_pic = [torch.randint(0, 256, (n, h, w, c), dtype=torch.uint8, device=dev) for _ in range(nb)]
    nv_full = [torch.randint(0, 256, (n, 3 * Hf // 2, w), dtype=torch.uint8, device=dev) for _ in range(nb)]
    nv_pic = [torch.randint(0, 256, (n, 3 * h // 2, w), dtype=torch.uint8, device=dev) for _ in range(nb)]
    us = {}
    timings = {
        'decode_u8_plain': lambda i: ops.stream_frame_in(rgb_pic[i], None, lrs[i], prev, hrp, s),
        'decode_u8_window': lambda i: ops.stream_frame_in(rgb_full[i], None, lrs[i], prev, hrp, s, window=(top, 0)),
        'decode_nv12_plain': lambda i: ops.stream_frame_in_yuv420(nv_pic[i], 'nv12', None, lrs[i], prev, hrp, s),
        'decode_nv12_window': lambda i: ops.stream_frame_in_yuv(nv_full[i], 'nv12', 'bt601', None, lrs[i], prev, hrp,
                                                                s, window=(top, 0)),
    }
    for k, fn in timings.items():
        us[k] = bench._time_graph(fn, nb, reps, torch) * 1e6
    del rgb_full, rgb_pic, nv_full, nv_pic
    hrs = [torch.rand(n, c, H, W, device=dev) for _ in range(nb)]
    u8s = [torch.empty(n, H, W, c, dtype=torch.uint8, device=dev) for _ in range(nb)]
    pads = [torch.empty(n, s * Hf, W, c, dtype=torch.uint8, device=dev) for _ in range(nb)]
    nvs = [torch.empty(n, 3 * H // 2, W, dtype=torch.uint8, device=dev) for _ in range(nb)]
    nv_pads = [torch.empty(n, 3 * s * Hf // 2, W, dtype=torch.uint8, device=dev) for _ in range(nb)]
    y0 = (s * Hf - H) // 2 // 2 * 2
    timings = {
        'to_uint8_plain': lambda i: ops.float_to_uint8_nhwc(hrs[i], u8s[i]),
        'to_uint8_window': lambda i: ops.float_to_uint8_nhwc_window(hrs[i], pads[i], (y0, 0)),
        'encode_nv12_plain': lambda i: ops.rgb_u8_to_yuv420(u8s[i], 'nv12', out=nvs[i]),
        'encode_nv12_window': lambda i: ops.rgb_to_yuv('nv12', 'bt601', rgb_u8=u8s[i], out=nv_pads[i],
                                                       window=(y0, 0)),
    }
    for k, fn in timings.items():
        us[k] = bench._time_graph(fn, nb, reps, torch) * 1e6
    line = {
        'metric': 'hr_frames_per_sec_4xBD_letterbox_134x320_in_180x320', 'unit': 'frames/s',
        'device': torch.cuda.get_device_name(0), 'power_limit_w': power_limit_w(),
        'clips': n, 'frames_per_clip': t, 'chunk': chunk, 'reps': args.reps,
        'results': {k: {'median': statistics.median(v), 'min': min(v), 'max': max(v), 'runs': v}
                    for k, v in runs.items()},
        'crop_out_frame_identical_to_precropped_placed': identical,
        'launches_per_step': launches,
        'kernel_us': us,
    }
    print(json.dumps(line), flush=True)


def _graph_us(fn, launches=20, reps=50):
    """Mean time of fn (enqueues on the current stream) over `reps` replays of a graph of `launches` calls."""
    import torch
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(launches):
            fn()
    g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (reps * launches)


def pad_bench(args):
    import numpy as np
    import torch
    import bench
    import tecogan_b200 as T
    ops = sys.modules['tecogan-pytorch_b200.ops']
    L = sys.modules['tecogan-pytorch_b200.lib']
    assert torch.cuda.is_available(), 'stream_bench.py needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    bench.select_workload('bd4')
    n, (c, h, w), s = bench.CLIPS_PER_GPU, bench.LR, bench.SCALE
    t, p = args.frames, 5
    net = T.FRNet(3, 3, 64, 10, 'BD', s)
    net.load_state_dict(bench.make_params(), strict=True)
    net = net.to(dev).eval()
    to_u8 = lambda x: np.ascontiguousarray(np.rint(x * 255.0).astype(np.uint8).transpose(0, 1, 3, 4, 2))   # noqa
    u8 = torch.from_numpy(to_u8(bench.synthetic_clips(n, t, seed=100).numpy())).pin_memory()
    shots = [bench.synthetic_clips(n, 32, seed=200 + i).numpy() for i in range(-(-t // 32))]
    cut_u8 = torch.from_numpy(to_u8(np.concatenate(shots, axis=1)[:, :t])).pin_memory()
    arms = {'plain': (u8, {}), 'pad5': (u8, dict(pad_front=p)),
            'plain_cuts32': (cut_u8, dict(scene_cut=10.0)), 'pad5_cuts32': (cut_u8, dict(scene_cut=10.0, pad_front=p))}
    opened = {k: net.stream(n, h, w, device=dev, **kw) for k, (_, kw) in arms.items()}
    runs = {k: [] for k in arms}
    cuts = {k: 0 for k in arms}
    for rep in range(args.reps + 1):                   # rep 0: untimed warm-up (graph capture)
        for k, (src, _) in arms.items():
            st = opened[k]
            found = 0
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(0, t, 16):
                st.push(src[:, i:i + 16])
                if st.scene_cut is not None:
                    found += int(st.last_cuts.sum())
            st.flush()
            if st.scene_cut is not None:
                found += int(st.last_cuts.sum())
            torch.cuda.synchronize()
            fps = n * t / (time.perf_counter() - t0)
            if rep:
                runs[k].append(fps)
                cuts[k] = found
    eng = opened['pad5']._engine
    warm_n = _graph_us(lambda: eng._enqueue_warm(0), launches=1)
    one = net.stream(1, h, w, device=dev, pad_front=p)
    one.push(u8[:1, :1])
    e1 = one._engine
    warm_1 = _graph_us(lambda: e1._enqueue_warm(0), launches=1)
    ring = eng.ring
    lr, prev, hr, wh = eng.lr[0].clone(), eng.lr[1].clone(), eng.hr[1].clone(), eng.whr[0].clone()
    tabs = {'keep': [0] * n + [L.GATHER_KEEP] * n + [-1] * n, 'load': [0] * n + [L.GATHER_LOAD] * n + [1] * n}
    gather = {}
    nlr, nhr = n * c * h * w * 4, n * c * h * w * s * s * 4
    for k, v in tabs.items():
        tab = torch.tensor(v, dtype=torch.int32, device=dev)
        us = _graph_us(lambda: ops.stream_gather(ring, tab, wh, lr, prev, hr, s))
        nbytes = 2 * nlr if k == 'keep' else 4 * nlr + 2 * nhr
        gather[k] = dict(us=round(us, 2), bytes=nbytes, tb_per_s=round(nbytes / us / 1e6, 3))
    for st in list(opened.values()) + [one]:
        st.close()
    med = {k: round(statistics.median(v), 1) for k, v in runs.items()}
    print(json.dumps({
        'metric': 'hr_frames_per_sec_4xBD_pad5', 'gpu': torch.cuda.get_device_name(dev), 'power_limit_w': power_limit_w(),
        'frames': t, 'reps': args.reps, 'push': 16, 'median': med,
        'runs': {k: [round(x, 1) for x in v] for k, v in runs.items()}, 'cuts_reported': cuts,
        'cuts_expected': n * (-(-t // 32) - 1),
        'warm_step_us': {'batch_n': round(warm_n, 1), 'batch_1': round(warm_1, 1)},
        'warm_start_us': {'batch_n': round(p * warm_n, 1), 'batch_1': round(p * warm_1, 1)},
        'gather_per_step': gather}))


def insize_bench(args):
    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import bench
    import tecogan_b200 as T
    from oracle import yuv_oracle as Y
    assert torch.cuda.is_available(), 'stream_bench.py needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    bench.select_workload('bd4')
    t, k = args.frames, 16
    net = T.FRNet(3, 3, 64, 10, 'BD', bench.SCALE)
    net.load_state_dict(bench.make_params(), strict=True)
    net = net.to(dev).eval()
    rng = np.random.default_rng(7)

    def source(n, h, w):
        """n x k smooth RGB frames (noise upsampled 8x, shifted a pixel a frame) as pinned NV12 [n,k,3h/2,w]."""
        base = rng.integers(0, 256, (n, h // 8 + 1, w // 8 + 2, 3)).astype(np.uint8)
        big = np.repeat(np.repeat(base, 8, 1), 8, 2)
        rgb = np.stack([big[:, :h, i:i + w] for i in range(k)], 1)
        return torch.from_numpy(Y.rgb_to_yuv420(np.ascontiguousarray(rgb), 'nv12')).pin_memory()

    arms, opened, frames = {}, {}, {}
    for n in (1, 2):
        frames[n] = (source(n, 1080, 1920), source(n, 540, 960))
        arms[f'insize_1080p_n{n}'] = (n, 0, dict(in_size=(540, 960)))
        arms[f'direct_540p_n{n}'] = (n, 1, {})
    for name, (n, i, kw) in arms.items():
        h, w = (1080, 1920) if i == 0 else (540, 960)
        opened[name] = net.stream(n, h, w, device=dev, input='nv12', out_format='nv12', **kw)
    runs = {name: [] for name in arms}
    for rep in range(args.reps + 1):                   # rep 0: untimed warm-up (graph capture)
        for name, (n, i, _) in arms.items():
            st, src = opened[name], frames[n][i]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(0, t, k):
                out = st.push(src, out='device')
            torch.cuda.synchronize()
            fps = n * t / (time.perf_counter() - t0)
            assert tuple(out.shape) == (n, k, 3240, 3840)
            if rep:
                runs[name].append(fps)
    launches = {name: st._engine.launches_per_step for name, st in opened.items()}
    frame_in = {}
    for name, (n, i, _) in arms.items():
        st, src = opened[name], frames[n][i]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st.push(src, out='device')
            torch.cuda.synchronize()
        kern = 'frame_in_resample_kernel' if i == 0 else 'stream_frame_in_kernel'
        evs = [e for e in prof.events() if e.device_type.name == 'CUDA' and kern in e.name]
        us = sum(e.time_range.elapsed_us() for e in evs) / len(evs) if evs else float("nan")
        h, w = (1080, 1920) if i == 0 else (540, 960)
        nbytes = n * (h * w * 3 // 2 + 3 * 540 * 960 * 4)
        frame_in[name] = dict(kernel=kern, launches=len(evs), us=round(us, 2), bytes=nbytes,
                              tb_per_s=round(nbytes / us / 1e6, 3))
    for st in opened.values():
        st.close()
    print(json.dumps({
        'metric': 'hr_frames_per_sec_4xBD_nv12_1080p_insize_540x960', 'gpu': torch.cuda.get_device_name(dev),
        'power_limit_w': power_limit_w(), 'frames': t, 'reps': args.reps, 'push': k,
        'median': {name: round(statistics.median(v), 1) for name, v in runs.items()},
        'runs': {name: [round(x, 1) for x in v] for name, v in runs.items()}, 'launches_per_step': launches,
        'frame_in_per_step': frame_in}))




def yuv422_10_bench(args):
    """The 10-bit 4:2:2 arms at bench.py's bd4 shape: k = 16 pushes of pinned frames, in and out of one layout, next to
    RGB and P010 (BT.709) in the same run, the arms alternating in every rep (rep 0 an untimed warm-up); then each
    layout's frame-input decode and fp32 encode alone, CUDA-graph timed over 8 rotating buffer sets."""
    import numpy as np
    import torch
    import bench
    import tecogan_b200 as T
    from oracle import yuv_color as C
    from oracle import yuv_422_10 as V
    ops = sys.modules['tecogan-pytorch_b200.ops']
    assert torch.cuda.is_available(), 'stream_bench.py needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    bench.select_workload('bd4')
    n, (c, h, w), s = bench.CLIPS_PER_GPU, bench.LR, bench.SCALE
    t, H, W = args.frames, s * h, s * w
    net = T.FRNet(3, 3, 64, 10, 'BD', s)
    net.load_state_dict(bench.make_params(), strict=True)
    net = net.to(dev).eval()
    clips = bench.synthetic_clips(n, t, seed=100).numpy().transpose(0, 1, 3, 4, 2)     # [n,t,h,w,c] in [0,1]
    u8 = np.ascontiguousarray(np.rint(clips * 255.0).astype(np.uint8))
    rgb10 = V.quantize10(clips)
    samples = V.encode_samples(rgb10, 'bt709')
    sources = {'rgb': (u8, {}),
               'p010_709': (C.rgb_to_yuv(rgb10, 'p010', 'bt709'), dict(input='p010', out_format='p010'))}
    for lay in V.LAYOUTS:
        sources[f'{lay}_709'] = (V.join_planes(*samples, lay), dict(input=lay, out_format=lay))
    pins = {k: torch.from_numpy(f).pin_memory() for k, (f, _) in sources.items()}
    opened = {k: net.stream(n, h, w, device=dev, **kw, **({'in_color': 'bt709', 'out_color': 'bt709'} if kw else {}))
              for k, (_, kw) in sources.items()}
    runs = {k: [] for k in sources}
    outputs = {}
    for rep in range(args.reps + 1):
        for k in sources:
            opened[k].reset(range(n))
            outputs[k] = None
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            outputs[k] = [opened[k].push(pins[k][:, i:i + 16]) for i in range(0, t, 16)]
            torch.cuda.synchronize()
            if rep:
                runs[k].append(n * t / (time.perf_counter() - t0))
    launches = {k: st._engine.launches_per_step for k, st in opened.items()}
    for st in opened.values():
        st.close()
    got = {k: np.concatenate(v, axis=1) for k, v in outputs.items()}
    # P210: frame by frame the oracle's encode of the fp32 HR frames of a device loop of FRNet.step over its decode;
    # I422_10 and v210: the same samples as P210
    identical = {}
    lr = torch.from_numpy(V.yuv_to_rgb(sources['p210_709'][0], 'p210', 'bt709').astype(np.float32) / np.float32(1023))
    lr = lr.permute(0, 1, 4, 2, 3).contiguous()
    ok = got['p210_709'].shape == (n, t, 2 * H, W)
    lr_prev, hr_prev = torch.zeros(n, c, h, w, device=dev), torch.zeros(n, c, H, W, device=dev)
    with torch.no_grad():
        for i in range(t):
            if not ok:
                break
            cur = lr[:, i].to(dev)
            hr_prev = net.step(cur, lr_prev, hr_prev)
            lr_prev = cur
            ok = np.array_equal(got['p210_709'][:, i], V.rgb_f32_to_yuv(hr_prev.permute(0, 2, 3, 1).cpu().numpy(),
                                                                        'p210', 'bt709'))
    identical['p210_709'] = bool(ok)
    ref = V.split_planes(got['p210_709'], 'p210')
    for lay in ('i422_10', 'v210'):
        identical[f'{lay}_709'] = all(np.array_equal(a, b) for a, b in zip(V.split_planes(got[f'{lay}_709'], lay, W),
                                                                           ref))
    del got, outputs
    # the kernels alone: 8 rotating sets of 4 frames
    nb, reps = 8, 60
    lrs = [torch.empty(n, c, h, w, device=dev) for _ in range(nb)]
    prev, hrp = torch.empty(n, c, h, w, device=dev), torch.empty(n, c, H, W, device=dev)
    hrs = [torch.rand(n, c, H, W, device=dev) for _ in range(nb)]
    decode, encode, decode_bytes, encode_bytes = {}, {}, {}, {}
    for lay in ('p010',) + V.LAYOUTS:
        shape = (n, *((3 * h // 2, w) if lay == 'p010' else V.frame_shape(lay, h, w)))
        dt = ops.yuv_word_dtype(lay)
        src = [torch.randint(0, 256, shape, dtype=torch.uint8, device=dev) if dt == torch.uint8 else
               torch.randint(0, 1 << 15, shape, dtype=torch.int16, device=dev).view(torch.uint16) for _ in range(nb)]
        sec = bench._time_graph(lambda i: ops.stream_frame_in_yuv(src[i], lay, 'bt709', None, lrs[i], prev, hrp, s),
                                nb, reps, torch)
        decode[lay] = sec * 1e6
        decode_bytes[lay] = src[0].numel() * src[0].element_size() + n * c * h * w * 4
        oshape = (n, *((3 * H // 2, W) if lay == 'p010' else V.frame_shape(lay, H, W)))
        outs = [torch.empty(oshape, dtype=dt, device=dev) for _ in range(nb)]
        sec = bench._time_graph(lambda i: ops.rgb_to_yuv(lay, 'bt709', rgb_f32=hrs[i], out=outs[i]), nb, reps, torch)
        encode[lay] = sec * 1e6
        encode_bytes[lay] = n * c * H * W * 4 + outs[0].numel() * outs[0].element_size()
        del src, outs
    line = {
        'metric': 'hr_frames_per_sec_4xBD_3x134x320_streamed_yuv422_10', 'unit': 'frames/s',
        'device': torch.cuda.get_device_name(0), 'power_limit_w': power_limit_w(), 'sm_clock_mhz': sm_clock_mhz(),
        'clips': n, 'frames_per_clip': t, 'reps': args.reps, 'chunk': 16,
        'results': {k: {'median': statistics.median(v), 'min': min(v), 'max': max(v), 'runs': v}
                    for k, v in runs.items()},
        'identical': identical,
        'launches_per_step': launches,
        'decode_us': decode, 'decode_bytes_per_step': decode_bytes,
        'decode_tb_per_s': {k: decode_bytes[k] / v * 1e-6 for k, v in decode.items()},
        'encode_us': encode, 'encode_bytes_per_step': encode_bytes,
        'encode_tb_per_s': {k: encode_bytes[k] / v * 1e-6 for k, v in encode.items()},
    }
    print(json.dumps(line), flush=True)


def sm_clock_mhz():
    try:
        r = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=clocks.sm,clocks.max.sm', '--format=csv,noheader,nounits'],
                           capture_output=True, text=True, timeout=20)
        return [float(v) for v in r.stdout.strip().splitlines()[0].split(',')]
    except Exception:
        return None


if __name__ == '__main__':
    main()
