"""Clip streaming engine: n lock-stepped clips through the FRNet recurrence with static device
buffers, one CUDA graph per ping-pong parity, pinned host staging and copy streams.

Replaces the per-frame host loop of FRNet.infer_sequence (reference tecogan_nets.py:269-281):
the reference does an H2D copy, ~60 library launches, a device sync, a D2H copy and a NumPy
uint8 conversion per frame; here a frame is one graph replay, the uint8/HWC conversion is a
kernel (tg_float_to_uint8_nhwc) and the copies overlap compute on side streams.
"""
import collections
import math
import numbers
import os
import weakref

import numpy as np
import torch

from . import ops


def _use_graph():
    return os.environ.get('TECOGAN_B200_GRAPH', '1') != '0'


class ClipEngine:
    def __init__(self, net, n, c, h, w, device, use_graph=None):
        # weak reference: the engine cache below must not keep a dropped net (and its graphs) alive
        self._net = weakref.ref(net)
        self.n, self.c, self.h, self.w = n, c, h, w
        self.device = torch.device(device)
        s = net.scale
        self.H, self.W = s * h, s * w
        dev = self.device
        with torch.cuda.device(dev):
            self.lr = [torch.zeros(n, c, h, w, device=dev) for _ in range(2)]
            self.hr = [torch.zeros(n, c, self.H, self.W, device=dev) for _ in range(2)]
            self.u8 = [torch.empty(n, self.H, self.W, c, dtype=torch.uint8, device=dev) for _ in range(2)]
            self.use_graph = _use_graph() if use_graph is None else use_graph
            self.graphs = [None, None]
            self.main = torch.cuda.Stream(device=dev)
            self.h2d = torch.cuda.Stream(device=dev)
            self.d2h = torch.cuda.Stream(device=dev)
            self.launches_per_step = None
            self.stage = None
            if self.use_graph:
                self._capture()

    @property
    def net(self):
        net = self._net()
        if net is None:
            raise ops.L.TecoganB200Error('ClipEngine: the FRNet it was built for has been deleted')
        return net

    def close(self):
        """Drop the CUDA graphs (and their private memory pool) and the static buffers."""
        self.graphs = [None, None]
        self.lr = self.hr = self.u8 = []
        self.stage = None

    # one frame: parity p consumes lr[p] (current), lr[p^1] (previous), hr[p^1] -> hr[p], u8[p]
    def _enqueue(self, p):
        # float32_to_uint8 + CHW->HWC happen inside the step (fused SRNet tail, or one extra kernel)
        self.net.step_into(self.lr[p], self.lr[p ^ 1], self.hr[p ^ 1], self.hr[p], out_u8=self.u8[p])

    def _capture(self):
        with torch.cuda.device(self.device):
            warm = torch.cuda.Stream(device=self.device)
            warm.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(warm):
                for p in (0, 1):            # builds packed weights, sets kernel attributes
                    self._enqueue(p)
            torch.cuda.current_stream().wait_stream(warm)
            torch.cuda.synchronize(self.device)
            pool = None
            for p in (0, 1):
                g = torch.cuda.CUDAGraph()
                before = ops.LAUNCH_COUNT
                with torch.cuda.graph(g, pool=pool):
                    self._enqueue(p)
                self.launches_per_step = ops.LAUNCH_COUNT - before
                pool = g.pool()
                self.graphs[p] = g
            self.reset()

    def reset(self):
        """lr_prev = hr_prev = 0 (reference tecogan_nets.py:269-270)."""
        with torch.cuda.device(self.device):
            for t in self.lr + self.hr:
                t.zero_()

    def run_frame(self, p):
        """Enqueue frame with parity p on the current stream."""
        if self.graphs[p] is not None:
            self.graphs[p].replay()
        else:
            before = ops.LAUNCH_COUNT
            self._enqueue(p)
            self.launches_per_step = ops.LAUNCH_COUNT - before

    def run_clips(self, lr_host, out_host=None):
        """lr_host: pinned CPU tensor (or CUDA tensor) [n,t,c,h,w] fp32; returns a pinned uint8
        tensor [t,n,H,W,c].  Three streams: H2D copies land in a 2-deep device staging ring (so the
        copy of frame i+1 overlaps the compute of frame i -- lr[p] itself is still being read as
        lr_prev), the main stream moves staging -> lr[p] (device-to-device, ~2 us) and replays the
        step graph, and the D2H stream drains the uint8 frames; one synchronisation at the end."""
        t = lr_host.shape[1]
        if out_host is None:   # caching host allocator: cheap after the first call
            out_host = torch.empty((t, self.n, self.H, self.W, self.c), dtype=torch.uint8,
                                   pin_memory=True)
        with torch.cuda.device(self.device):
            if self.stage is None:
                self.stage = [torch.empty_like(self.lr[0]) for _ in range(2)]
            self.main.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self.main):
                self.reset()
            staged = [None, None]          # H2D into stage[q] finished
            consumed = [None, None]        # stage[q] copied into lr[] (free for the next H2D)
            out_copied = [None, None]      # D2H of u8[p] finished
            self.h2d.wait_stream(self.main)
            for i in range(t):
                p = q = i & 1
                with torch.cuda.stream(self.h2d):
                    if consumed[q] is not None:
                        self.h2d.wait_event(consumed[q])
                    for k in range(self.n):
                        self.stage[q][k].copy_(lr_host[k, i], non_blocking=True)
                    staged[q] = torch.cuda.Event()
                    staged[q].record(self.h2d)
                with torch.cuda.stream(self.main):
                    self.main.wait_event(staged[q])
                    self.lr[p].copy_(self.stage[q], non_blocking=True)
                    consumed[q] = torch.cuda.Event()
                    consumed[q].record(self.main)
                    if out_copied[p] is not None:
                        self.main.wait_event(out_copied[p])    # u8[p] free to overwrite
                    self.run_frame(p)
                    done = torch.cuda.Event()
                    done.record(self.main)
                with torch.cuda.stream(self.d2h):
                    self.d2h.wait_event(done)
                    out_host[i].copy_(self.u8[p], non_blocking=True)
                    out_copied[p] = torch.cuda.Event()
                    out_copied[p].record(self.d2h)
            self.d2h.synchronize()
            self.main.synchronize()
        return out_host


# Engines are cached per net (weakly: deleting the net frees its engines) and per clip geometry,
# least-recently-used first; at most TECOGAN_B200_MAX_ENGINES (default 3) geometries per net stay
# captured -- each holds two CUDA graphs and their pool (hundreds of MB to a few GB at video sizes).
_ENGINES = weakref.WeakKeyDictionary()


def _max_engines():
    return max(1, int(os.environ.get('TECOGAN_B200_MAX_ENGINES', '3')))


def _param_signature(net):
    p = next(net.parameters())
    return (str(p.device), p.data_ptr())


def get_engine(net, n, c, h, w, device):
    per_net = _ENGINES.get(net)
    sig = _param_signature(net)
    if per_net is None or per_net['sig'] != sig:
        # first use, or the parameters moved (net.to(other device) / re-materialised): captured graphs
        # would read freed buffers -> drop every engine of this net
        if per_net is not None:
            for eng in per_net['lru'].values():
                eng.close()
        per_net = _ENGINES[net] = {'sig': sig, 'lru': collections.OrderedDict()}
    lru = per_net['lru']
    key = (n, c, h, w, str(device))
    eng = lru.get(key)
    if eng is None:
        while len(lru) >= _max_engines():
            lru.popitem(last=False)[1].close()
        eng = lru[key] = ClipEngine(net, n, c, h, w, device)
    else:
        lru.move_to_end(key)
        # parameters may have changed since capture: repack in place (graphs read the same buffers)
        net.refresh_packed_weights()
    return eng


def release_engines(net=None):
    """Free the cached engines of `net` (all nets when None)."""
    nets = [net] if net is not None else list(_ENGINES.keys())
    for k in nets:
        per_net = _ENGINES.pop(k, None)
        if per_net is not None:
            for eng in per_net['lru'].values():
                eng.close()


def infer_clips(net, lr_data, device):
    """lr_data [n,t,c,h,w] fp32 (CPU or CUDA) -> np.uint8 [n,t,H,W,c]."""
    if lr_data.dim() != 5:
        raise ValueError('infer_clips expects ntchw')
    n, t, c, h, w = lr_data.shape
    device = torch.device(device)
    if device.type != 'cuda':
        raise ops.L.TecoganB200Error('tecogan-b200 runs on CUDA devices only (no CPU path)')
    eng = get_engine(net, n, c, h, w, device)
    src = lr_data.detach()
    if src.dtype != torch.float32:
        src = src.float()
    if not src.is_cuda and not src.is_pinned():
        src = src.pin_memory()           # pageable input: one staging copy (pass pinned to avoid)
    out = eng.run_clips(src)
    return out.numpy().transpose(1, 0, 2, 3, 4)


class StreamEngine(ClipEngine):
    """ClipEngine's static buffers, streams and per-parity step graphs, with the recurrent state (lr[p^1],
    hr[p^1], the parity) kept between calls of `run`, for video that arrives in chunks.  Like ClipEngine it holds
    its net weakly; VideoStream (FRNet.stream) holds the strong reference.

    Each graph starts with tg_stream_frame_in: it decodes the uint8 HWC frames of inp[p] into lr[p] (fp32 input:
    the caller copied lr[p], the kernel only resets) and zeroes lr[p^1][k] / hr[p^1][k] of the slots flagged in
    the device mask mask[p] -- the reset of one slot happens inside the captured step, and one graph serves every
    pattern of resets.  The step itself is the unchanged net.step_into.

    YUV input (yuv_in = 'nv12' / 'i420' / 'p010' / 'i420_10', or the 4:2:2 / 4:4:4 'yuy2' / 'uyvy' / 'i444' /
    'i444_10'): inp[p] holds [n,3h/2,w] frames ([n,h,2w] for 4:2:2, [n,3h,w] for 4:4:4; uint16 for the 10-bit
    layouts) and the first launch is tg_stream_frame_in_yuv420 (8 bit, BT.601 limited range: cv2's
    conversion) or tg_stream_frame_in_yuv (any other layout or colour) instead, with the same reset.  YUV output
    (yuv_out): each graph ends with the encode into yuv[p] [n,3H/2,W] (or that layout's shape) --
    tg_rgb_u8_to_yuv420 of u8[p] (8 bit,
    BT.601 limited range), tg_rgb_to_yuv of u8[p] (8 bit, other colours) or tg_rgb_to_yuv of the fp32 HR frame
    hr[p] (10 bit, uint16 yuv[p]) -- and the copies out read yuv[p] instead of u8[p].

    Resized output (out_size = (Ho, Wo)): the step runs without its uint8 output (nothing would read it) and is
    followed by tg_resample_nchw_f32 of the fp32 HR frame hr[p] into rs[p] -- uint8 [n,Ho,Wo,c], or fp32 [n,c,Ho,Wo]
    when a 10-bit encode follows -- with the per-axis tables built once (tables[0] rows, tables[1] columns).  The
    encode then reads rs[p] instead of u8[p] / hr[p], and the copies out read rs[p] (or yuv[p]).

    Scene cuts (scene_cut = threshold): after the frame input, tg_scene_cut scores lr[p] against lr[p^1] for every
    slot (the caller's resets of mask[p] score 0) into score[p] / cut[p], updating the per-slot state prev_mafd, and
    a second tg_stream_frame_in, reset-only with cut[p] as its mask, zeroes lr[p^1][k] / hr[p^1][k] of the slots
    with a detected cut -- the restart a reset of that slot at this frame would have made.  score[p] (float64 [n])
    and cut[p] (int32 [n]) are views of one int32 buffer rep[p] [3n], copied after each replay into the push's
    report [k,3n] (one device-to-device copy per frame).

    Copies overlap compute as in ClipEngine.run_clips.  uint8 input: inp[p] is itself the 2-deep staging ring (the
    step of parity p^1 never reads it), so the H2D of frame i+1 lands directly in the graph's input while frame i
    runs.  fp32 input: lr[p] is still read as lr_prev by frame i, so frames are staged as in run_clips."""

    def __init__(self, net, n, c, h, w, device, u8_input=True, bgr=False, yuv_in=None, yuv_out=None,
                 in_color='bt601', out_color='bt601', out_size=None, resize_filter='bicubic', scene_cut=None):
        dev = torch.device(device)
        self.u8_input, self.bgr = u8_input or yuv_in is not None, bgr
        self.yuv_in, self.yuv_out = yuv_in, yuv_out          # None or one of ops.YUV_LAYOUTS
        self.in_color, self.out_color = in_color, out_color
        self.mask = [torch.zeros(n, dtype=torch.int32, device=dev) for _ in range(2)]
        frame = ops.yuv_frame_shape(yuv_in, h, w) if yuv_in else (h, w, c)
        # 10-bit words: zeroed as int16, the same bits
        in_dtype = torch.int16 if yuv_in and ops.yuv_depth(yuv_in) == 10 else torch.uint8
        self.inp = ([torch.zeros(n, *frame, dtype=in_dtype, device=dev).view(_word_dtype(yuv_in)) for _ in range(2)]
                    if self.u8_input else None)
        H, W = net.scale * h, net.scale * w
        self.out_size = tuple(out_size) if out_size else None
        Ho, Wo = self.out_size or (H, W)
        self.tables, self.rs = None, None
        if self.out_size:
            self.tables = [tuple(t.to(dev) for t in ops.resample_table(a, b, resize_filter))
                           for a, b in ((H, Ho), (W, Wo))]
            f32 = yuv_out is not None and ops.yuv_depth(yuv_out) == 10
            self.rs = [torch.empty((n, c, Ho, Wo) if f32 else (n, Ho, Wo, c),
                                   dtype=torch.float32 if f32 else torch.uint8, device=dev) for _ in range(2)]
        self.yuv = ([torch.empty(n, *ops.yuv_frame_shape(yuv_out, Ho, Wo), dtype=_word_dtype(yuv_out), device=dev)
                     for _ in range(2)]
                    if yuv_out else None)
        self.scene_cut = scene_cut
        self.prev_mafd = self.work = self.rep = self.score = self.cut = None
        self.report = None               # [k,3n] int32 of the last run: score[p] / cut[p] after each frame
        self._report_dev = self._report_host = None
        if scene_cut is not None:
            self.prev_mafd = torch.full((n,), -1.0, dtype=torch.float64, device=dev)
            self.work = ops.scene_cut_work(n, dev)
            self.rep = [torch.zeros(3 * n, dtype=torch.int32, device=dev) for _ in range(2)]
            self.score = [r[:2 * n].view(torch.float64) for r in self.rep]
            self.cut = [r[2 * n:] for r in self.rep]
        self.sig = _param_signature(net)
        self.parity = 0                  # parity of the next frame
        self.mask_set = [False, False]   # mask[p] holds a reset pattern (cleared before the next replay)
        self.in_free = [None, None]      # event: the replay that last read inp[p] / stage[p] finished
        self.out_copied = [None, None]   # event: the D2H of u8[p] (yuv[p]) finished
        # the capture's warm-up steps update prev_mafd; that state is never read, because the first push resets every
        # slot (VideoStream._pending) and a reset sets prev_mafd := -1 without reading it
        super().__init__(net, n, c, h, w, dev)     # lr / hr / u8, streams, the two graphs of _enqueue below

    def close(self):
        super().close()
        self.mask, self.inp, self.yuv = [], None, None
        self.tables, self.rs = None, None
        self.prev_mafd = self.work = self.rep = self.score = self.cut = self.report = None
        self._report_dev = self._report_host = None

    def _enqueue(self, p):
        if self.yuv_in in YUV420 and self.in_color == 'bt601':
            ops.stream_frame_in_yuv420(self.inp[p], self.yuv_in, self.mask[p], self.lr[p], self.lr[p ^ 1],
                                       self.hr[p ^ 1], self.net.scale)
        elif self.yuv_in:
            ops.stream_frame_in_yuv(self.inp[p], self.yuv_in, self.in_color, self.mask[p], self.lr[p],
                                    self.lr[p ^ 1], self.hr[p ^ 1], self.net.scale)
        else:
            ops.stream_frame_in(self.inp[p] if self.u8_input else None, self.mask[p], self.lr[p], self.lr[p ^ 1],
                                self.hr[p ^ 1], self.net.scale, self.bgr)
        if self.scene_cut is not None:
            ops.scene_cut(self.lr[p], self.lr[p ^ 1], self.mask[p], self.scene_cut, self.prev_mafd, self.work,
                          self.score[p], self.cut[p])
            # a detected cut restarts the slot: the reset-only frame input with cut[p] as its mask
            ops.stream_frame_in(None, self.cut[p], self.lr[p], self.lr[p ^ 1], self.hr[p ^ 1], self.net.scale)
        if self.out_size is None:
            super()._enqueue(p)
            rgb_u8, rgb_f32 = self.u8[p], self.hr[p]
        else:
            self.net.step_into(self.lr[p], self.lr[p ^ 1], self.hr[p ^ 1], self.hr[p], out_u8=None)
            f32 = self.rs[p].dtype == torch.float32
            ops.resample(self.hr[p], *self.tables, out_u8=None if f32 else self.rs[p], out_f32=self.rs[p] if f32 else None)
            rgb_u8 = rgb_f32 = self.rs[p]
        if self.yuv_out in YUV420 and self.out_color == 'bt601':
            ops.rgb_u8_to_yuv420(rgb_u8, self.yuv_out, out=self.yuv[p])
        elif self.yuv_out and ops.yuv_depth(self.yuv_out) == 8:
            ops.rgb_to_yuv(self.yuv_out, self.out_color, rgb_u8=rgb_u8, out=self.yuv[p])
        elif self.yuv_out:
            # 10 bit: from the step's fp32 HR frame (or its resize), two more bits than the uint8 output keeps
            ops.rgb_to_yuv(self.yuv_out, self.out_color, rgb_f32=rgb_f32, out=self.yuv[p])

    def _set_mask(self, p, slots):
        """On the main stream, before the replay of parity p: mask[p] = 1 for `slots`, 0 elsewhere."""
        if slots:
            self.mask[p].zero_()
            for k in slots:
                self.mask[p][k].fill_(1)
            self.mask_set[p] = True
        elif self.mask_set[p]:
            self.mask[p].zero_()
            self.mask_set[p] = False

    def run(self, frames, reset_slots, out_host):
        """frames: uint8 [n,k,h,w,c] (u8_input), uint8 / uint16 [n,k,*yuv_frame_shape] (yuv_in) or fp32
        [n,k,c,h,w], each
        frame contiguous, pinned host or on this device.
        Slots in `reset_slots` start a new video at frame 0.  Returns uint8 [n,k,H,W,c] (or [n,k,3H/2,W] words with
        yuv_out; Ho, Wo instead of H, W with out_size): a pinned host tensor (out_host; one synchronisation, at the end) or a new tensor on the device,
        ordered on the current stream (no synchronisation)."""
        n, k = self.n, frames.shape[1]
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream()
            self.net.refresh_packed_weights()        # a load_state_dict between pushes takes effect
            for st in (self.main, self.h2d, self.d2h):
                st.wait_stream(cur)
            # what the step graph leaves for the copy out
            res = self.yuv if self.yuv_out else self.rs if self.out_size else self.u8
            shape = (n, k, *res[0].shape[1:])
            if out_host:
                out = torch.empty(shape, dtype=res[0].dtype, pin_memory=True)
            else:
                out = torch.empty(shape, dtype=res[0].dtype, device=self.device)
            report = None
            if self.scene_cut is not None:
                # kept between pushes (read on the current stream, which the next push's streams wait for)
                if self._report_dev is None or self._report_dev.shape[0] < k:
                    self._report_dev = torch.empty((max(k, 16), 3 * n), dtype=torch.int32, device=self.device)
                report = self._report_dev[:k]
            if not self.u8_input and self.stage is None:
                self.stage = [torch.empty_like(self.lr[0]) for _ in range(2)]
            dst = self.inp if self.u8_input else self.stage
            for i in range(k):
                p = self.parity
                with torch.cuda.stream(self.h2d):
                    if self.in_free[p] is not None:
                        self.h2d.wait_event(self.in_free[p])
                    for j in range(n):
                        dst[p][j].copy_(frames[j, i], non_blocking=True)
                    staged = torch.cuda.Event()
                    staged.record(self.h2d)
                with torch.cuda.stream(self.main):
                    self.main.wait_event(staged)
                    if not self.u8_input:
                        self.lr[p].copy_(self.stage[p], non_blocking=True)
                    self._set_mask(p, reset_slots if i == 0 else None)
                    if out_host and self.out_copied[p] is not None:
                        self.main.wait_event(self.out_copied[p])     # res[p] free to overwrite
                    self.run_frame(p)
                    if report is not None:
                        report[i].copy_(self.rep[p], non_blocking=True)
                    done = torch.cuda.Event()
                    done.record(self.main)
                    self.in_free[p] = done
                    if not out_host:
                        out[:, i].copy_(res[p], non_blocking=True)
                if out_host:
                    with torch.cuda.stream(self.d2h):
                        self.d2h.wait_event(done)
                        for j in range(n):
                            out[j, i].copy_(res[p][j], non_blocking=True)
                        self.out_copied[p] = torch.cuda.Event()
                        self.out_copied[p].record(self.d2h)
                self.parity ^= 1
            if out_host:
                if report is not None:       # the D2H stream has waited on the last replay's event
                    if self._report_host is None or self._report_host.shape[0] < k:
                        self._report_host = torch.empty(self._report_dev.shape, dtype=torch.int32, pin_memory=True)
                    with torch.cuda.stream(self.d2h):
                        self._report_host[:k].copy_(report, non_blocking=True)
                    report = self._report_host[:k]
                self.d2h.synchronize()   # after every replay (D2H waited on each) and so after every H2D
            else:
                cur.wait_stream(self.main)
                cur.wait_stream(self.h2d)    # a device input may be freed once the call returns
        self.report = report
        return out


YUV420 = ops.YUV420_LAYOUTS       # 'nv12', 'i420'
YUV = ops.YUV_LAYOUTS             # those, the 10-bit 'p010', 'i420_10', 4:2:2 'yuy2', 'uyvy', 4:4:4 'i444', 'i444_10'
_YUV_422_444 = ops.YUV422_LAYOUTS + ops.YUV444_LAYOUTS
COLORS = ops.YUV_COLORS           # 'bt601' (the default, cv2's conversion), 'bt709', 'bt601-full', 'bt709-full'


def _word_dtype(layout):
    return torch.uint16 if layout and ops.yuv_depth(layout) == 10 else torch.uint8


class VideoStream:
    """n lock-stepped video slots through FRNet with the recurrent state carried between `push` calls.
    Created by FRNet.stream(); see there."""

    def __init__(self, net, n, h, w, device=None, input='uint8', channel_order='rgb', out_format='rgb',
                 in_color='bt601', out_color='bt601', out_size=None, resize_filter='bicubic', scene_cut=None):
        if scene_cut is not None:
            scene_cut = _check_scene_cut(scene_cut)
        if input not in ('uint8', 'float32', *YUV):
            raise ValueError(f"input must be 'uint8', 'float32' or one of {YUV}, got {input!r}")
        if channel_order not in ('rgb', 'bgr'):
            raise ValueError(f"channel_order must be 'rgb' or 'bgr', got {channel_order!r}")
        if out_format not in ('rgb', *YUV):
            raise ValueError(f"out_format must be 'rgb' or one of {YUV}, got {out_format!r}")
        for arg, color, side in (('in_color', in_color, input), ('out_color', out_color, out_format)):
            if not isinstance(color, str) or color not in COLORS:
                raise ValueError(f'{arg} must be one of {COLORS}, got {color!r}')
            if side not in YUV and color != 'bt601':
                raise ValueError(f'{arg}={color!r} applies to YUV frames only, not to {side!r}')
        if input != 'uint8' and channel_order != 'rgb':
            raise ValueError(f"channel_order='bgr' applies to uint8 HWC input only, not input={input!r}")
        if not all(isinstance(v, int) and v > 0 for v in (n, h, w)):
            raise ValueError(f'n, h, w must be positive ints, got {(n, h, w)}')
        if not isinstance(resize_filter, str) or resize_filter not in ops.RESIZE_FILTERS:
            raise ValueError(f'resize_filter must be one of {ops.RESIZE_FILTERS}, got {resize_filter!r}')
        if out_size is None and resize_filter != 'bicubic':
            raise ValueError(f'resize_filter={resize_filter!r} applies to a resized stream only (give out_size)')
        if out_size is not None:
            out_size = _check_out_size(out_size, net.scale * h, net.scale * w, out_format)
        yuv = [f for f in (input, out_format) if f in YUV]
        for f in yuv:
            if f not in _YUV_422_444 and (h % 2 or w % 2):
                raise ValueError(f'{f} frames are YUV 4:2:0: h and w must be even, got {h}x{w}')
            if f in ops.YUV422_LAYOUTS and w % 2:
                raise ValueError(f'{f} frames are YUV 4:2:2: w must be even, got {h}x{w}')
        if yuv and net.fnet.in_nc != 3:
            raise ValueError(f'{yuv[0]} frames carry 3 colour channels, the net takes {net.fnet.in_nc}')
        device = torch.device('cuda') if device is None else torch.device(device)
        if device.type != 'cuda':
            raise ops.L.TecoganB200Error('tecogan-b200 runs on CUDA devices only (no CPU path)')
        self.net, self.n, self.h, self.w = net, n, h, w
        self.c = net.fnet.in_nc
        self.device, self.input, self.channel_order, self.out_format = device, input, channel_order, out_format
        self.in_color, self.out_color = in_color, out_color
        self.out_size, self.resize_filter = out_size, resize_filter
        self.scene_cut = scene_cut
        # the latest push's detected cuts (bool [n,k]) and scores (float64 [n,k]): NumPy after out='host', CUDA
        # tensors after out='device'; None before the first push and without scene_cut
        self.last_cuts = self.last_scores = None
        self._engine = None                  # built (graphs captured) by the first push
        self._pending = [True] * n           # a new stream starts every slot from zero state
        _check_inference(net)

    def reset(self, slots):
        """Mark `slots` (indices) to start a new video at the first frame of the next push."""
        for k in slots:
            if not 0 <= int(k) < self.n:
                raise IndexError(f'slot {k} out of range for a stream of {self.n} slots')
            self._pending[int(k)] = True

    def close(self):
        """Free the CUDA graphs and the device buffers; the stream cannot be pushed to afterwards."""
        if self._engine:
            self._engine.close()
        self._engine = False

    def push(self, frames, reset=None, out='host'):
        """Run the next k frames of every slot.

        frames: uint8 [n,k,h,w,c] (input='uint8'; [k,h,w,c] when n == 1), uint8 [n,k,3h/2,w] (input='nv12' or
                'i420'; [k,3h/2,w] when n == 1) or fp32 [n,k,c,h,w] (input='float32'; [k,c,h,w] when n == 1), each
                frame contiguous (a slice [:, i:i+k] of a clip is fine), as a torch tensor on the host (pinned or
                pageable) or on the stream's device, or a NumPy array.  Nothing is converted: another dtype,
                layout or size raises.
        reset:  n bools; slot k starts a new video at the first frame of this push (its recurrent state is zeroed,
                as for frame 0 of FRNet.infer_sequence).
        out:    'host' -> NumPy uint8 [n,k,H,W,c] (one synchronisation); 'device' -> a new CUDA uint8 tensor
                [n,k,H,W,c], ordered on the current stream (no synchronisation; a pinned host input must then
                stay unchanged until that stream has passed this push).  With out_format 'nv12' / 'i420' the
                frames are uint8 [n,k,3H/2,W] instead, with 'p010' / 'i420_10' uint16 [n,k,3H/2,W].  A stream
                opened with out_size=(Ho, Wo) returns Ho x Wo frames in place of H x W.
        10-bit input ('p010', 'i420_10') takes uint16 frames [n,k,3h/2,w] ([k,3h/2,w] when n == 1), torch.uint16 or
        NumPy uint16; uint8 frames into a 10-bit stream raise, and so do uint16 frames into an 8-bit one.
        4:2:2 and 4:4:4, in and out: 'yuy2' / 'uyvy' frames are uint8 [n,k,h,2w], 'i444' uint8 [n,k,3h,w] and
        'i444_10' uint16 [n,k,3h,w] (H, W or Ho, Wo on the output side).
        A stream opened with scene_cut=threshold restarts a slot at every detected cut, as reset= would have, and
        sets last_cuts (bool [n,k]) and last_scores (float64 [n,k]) for this push: NumPy with out='host', CUDA
        tensors ordered on the current stream with out='device'.  A reset requested by the caller scores 0 and is
        not reported as a cut.
        """
        if self._engine is False:
            raise ops.L.TecoganB200Error('VideoStream.push: the stream is closed')
        if out not in ('host', 'device'):
            raise ValueError(f"out must be 'host' or 'device', got {out!r}")
        frames = self._check_frames(frames)
        slots = list(self._pending)
        if reset is not None:
            reset = list(reset)
            if len(reset) != self.n:
                raise ValueError(f'reset has {len(reset)} entries, the stream has {self.n} slots')
            slots = [a or bool(b) for a, b in zip(slots, reset)]
        _check_inference(self.net)
        if self._engine is None:
            self._engine = self._build()
        elif _param_signature(self.net) != self._engine.sig:
            raise ops.L.TecoganB200Error('VideoStream.push: the net\'s parameters moved since the stream was '
                                         'built (net.to(...)?); open a new stream')
        if not frames.is_cuda and not frames.is_pinned():
            # pageable input: one staging copy of exactly this chunk (pass pinned memory to avoid it)
            frames = torch.empty(frames.shape, dtype=frames.dtype, pin_memory=True).copy_(frames)
        res = self._engine.run(frames, [k for k in range(self.n) if slots[k]], out == 'host')
        self._pending = [False] * self.n
        rep = self._engine.report
        if rep is not None:
            # [k,3n] int32: words [0,2n) the n float64 scores, [2n,3n) the n cut flags.  rep is the engine's report
            # buffer, reused by the next push, so the score words are copied into a new [k,2n] array first: a
            # slice's .contiguous() / ascontiguousarray is no copy when k == 1, and its row stride of 3n words
            # cannot be viewed as float64 for odd n.  On the device this runs on the current stream.
            n = self.n
            if out == 'host':
                r = rep.numpy()
                self.last_scores = r[:, :2 * n].copy(order='C').view(np.float64).T.copy()
                self.last_cuts = (r[:, 2 * n:] != 0).T.copy()
            else:
                words = torch.empty((rep.shape[0], 2 * n), dtype=torch.int32, device=rep.device)
                words.copy_(rep[:, :2 * n])
                self.last_scores = words.view(torch.float64).t().contiguous()
                self.last_cuts = (rep[:, 2 * n:] != 0).t().contiguous()
        return res.numpy() if out == 'host' else res

    def _check_frames(self, frames):
        L = ops.L
        if isinstance(frames, np.ndarray):
            if any(st < 0 for st in frames.strides):
                raise L.TecoganB200Error('VideoStream.push: each frame must be contiguous; got negative strides '
                                         '(cv2 [..., ::-1]: use channel_order="bgr" or np.ascontiguousarray)')
            frames = torch.from_numpy(frames)
        if not isinstance(frames, torch.Tensor):
            raise TypeError(f'VideoStream.push: frames must be a tensor or ndarray, got {type(frames).__name__}')
        dtype = torch.float32 if self.input == 'float32' else _word_dtype(self.input if self.input in YUV else None)
        if frames.dtype != dtype:
            raise L.TecoganB200Error(f'VideoStream.push: {self.input} stream expects {dtype} frames, got '
                                     f'{frames.dtype}')
        frame, layout = {'uint8': ((self.h, self.w, self.c), 'n,k,h,w,c'),
                         'float32': ((self.c, self.h, self.w), 'n,k,c,h,w')}.get(
                             self.input, (None, None))
        if frame is None:
            frame = ops.yuv_frame_shape(self.input, self.h, self.w)
            layout = ('n,k,h,2w' if self.input in ops.YUV422_LAYOUTS else
                      'n,k,3h,w' if self.input in ops.YUV444_LAYOUTS else 'n,k,3h/2,w')
        if frames.dim() == len(frame) + 1 and self.n == 1:
            frames = frames.unsqueeze(0)
        if (frames.dim() != len(frame) + 2 or frames.shape[0] != self.n or frames.shape[1] < 1
                or tuple(frames.shape[2:]) != frame):
            raise L.TecoganB200Error(f'VideoStream.push: frames {tuple(frames.shape)} do not match [{layout}] '
                                     f'with n={self.n}, {"x".join(map(str, frame))} per frame')
        if not frames[0, 0].is_contiguous():      # frames are copied one at a time: [n,k] may be a slice
            raise L.TecoganB200Error('VideoStream.push: each frame must be contiguous')
        if frames.is_cuda and frames.device != self._resolved_device():
            raise L.TecoganB200Error(f'VideoStream.push: frames on {frames.device}, the stream runs on '
                                     f'{self._resolved_device()}')
        if frames.requires_grad:
            raise L.TecoganB200Error('VideoStream.push: frames require grad (no backward exists for a stream)')
        return frames

    def _resolved_device(self):
        d = self.device
        return d if d.index is not None else torch.device('cuda', torch.cuda.current_device())

    def _build(self):
        if not torch.cuda.is_available():
            raise ops.L.TecoganB200Error('VideoStream: no CUDA device available (no CPU path)')
        dev = self._resolved_device()
        pdev = next(self.net.parameters()).device
        if pdev != dev:
            raise ops.L.TecoganB200Error(f'VideoStream: the net\'s parameters are on {pdev}, the stream runs on '
                                         f'{dev}; move the net first (net.to(device))')
        self.device = dev
        yuv_in = self.input if self.input in YUV else None
        yuv_out = self.out_format if self.out_format in YUV else None
        return StreamEngine(self.net, self.n, self.c, self.h, self.w, dev, u8_input=self.input == 'uint8',
                            bgr=self.channel_order == 'bgr', yuv_in=yuv_in, yuv_out=yuv_out,
                            in_color=self.in_color, out_color=self.out_color, out_size=self.out_size,
                            resize_filter=self.resize_filter, scene_cut=self.scene_cut)


def _check_scene_cut(threshold):
    """scene_cut -> float threshold, or ValueError: a real number (not a bool) in (0, 100]; NaN and inf refused."""
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real):
        raise ValueError(f'scene_cut must be None or a threshold in (0, 100], got {threshold!r}')
    t = float(threshold)
    if not (math.isfinite(t) and ops.scene_cut_threshold_ok(t)):
        raise ValueError(f'scene_cut threshold must be finite and in (0, 100], got {threshold!r}')
    return t


def _check_out_size(out_size, H, W, out_format):
    """out_size -> (Ho, Wo) ints, or ValueError: two positive ints within the resize's ratios of the H x W output,
    both even for a YUV 4:2:0 out_format, Wo even for 4:2:2."""
    if (not isinstance(out_size, (tuple, list)) or len(out_size) != 2
            or not all(isinstance(v, numbers.Integral) and not isinstance(v, bool) and v > 0 for v in out_size)):
        raise ValueError(f'out_size must be (Ho, Wo), two positive ints, got {out_size!r}')
    Ho, Wo = int(out_size[0]), int(out_size[1])
    if not (ops.resample_ratio_ok(H, Ho) and ops.resample_ratio_ok(W, Wo)):
        raise ValueError(f'out_size {Ho}x{Wo} from a {H}x{W} output: each axis must be within 1/4 to 2 times the '
                         f'output size')
    if out_format in YUV and out_format not in _YUV_422_444 and (Ho % 2 or Wo % 2):
        raise ValueError(f'{out_format} frames are YUV 4:2:0: out_size must be even, got {Ho}x{Wo}')
    if out_format in ops.YUV422_LAYOUTS and Wo % 2:
        raise ValueError(f'{out_format} frames are YUV 4:2:2: the width of out_size must be even, got {Ho}x{Wo}')
    return Ho, Wo


def _check_inference(net):
    if net.training and any(p.requires_grad for p in net.parameters()):
        raise ops.L.TecoganB200Error('FRNet.stream is inference only: call net.eval() (or set requires_grad=False '
                                     'on the parameters) first')
