"""Clip streaming engine: n lock-stepped clips through the FRNet recurrence with static device
buffers, one CUDA graph per ping-pong parity, pinned host staging and copy streams.

Replaces the per-frame host loop of FRNet.infer_sequence (reference tecogan_nets.py:269-281):
the reference does an H2D copy, ~60 library launches, a device sync, a D2H copy and a NumPy
uint8 conversion per frame; here a frame is one graph replay, the uint8/HWC conversion is a
kernel (tg_float_to_uint8_nhwc) and the copies overlap compute on side streams.
"""
import collections
import functools
import math
import numbers
import os
import weakref

import numpy as np
import torch

from . import ops


def _use_graph():
    return os.environ.get('TECOGAN_B200_GRAPH', '1') != '0'


def _record(stream):
    """A new event recorded on `stream`."""
    e = torch.cuda.Event()
    e.record(stream)
    return e


def _wait(stream, event):
    """`stream` waits for `event`; None: nothing to wait for."""
    if event is not None:
        stream.wait_event(event)


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
            self.in_free = [None, None]      # event: the staging buffer of parity p is free for the next H2D
            self.out_copied = [None, None]   # event: the D2H of parity p's output finished
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
            self.in_free = [None, None]
            self.out_copied = [None, None]
            self.h2d.wait_stream(self.main)
            for i in range(t):
                p = i & 1
                staged = self._stage(self.stage[p], lr_host[:, i], self.in_free[p])
                with torch.cuda.stream(self.main):
                    self.main.wait_event(staged)
                    self.lr[p].copy_(self.stage[p], non_blocking=True)
                    self.in_free[p] = _record(self.main)
                    done = self._step(p, True)
                self._drain(p, done, out_host[i], self.u8[p], True, per_slot=False)
            self._finish(None, True)
        return out_host

    # the copy pipeline of run_clips and the streams: H2D stream -> main stream -> D2H stream, one event per hand-over
    def _stage(self, dst, src, free):
        """On the H2D stream, once the event `free` (None: at once) has passed: dst[k] := src[k] for every slot.
        Returns the event of the copies."""
        with torch.cuda.stream(self.h2d):
            _wait(self.h2d, free)
            for k in range(self.n):
                dst[k].copy_(src[k], non_blocking=True)
            return _record(self.h2d)

    def _step(self, p, out_host, report=None):
        """On the current (main) stream: the step of parity p, after the D2H of its last output (host output), then the
        copy report = (dst, src) if given.  Returns the event of the step."""
        if out_host:
            _wait(self.main, self.out_copied[p])      # the output buffer is free to overwrite
        self.run_frame(p)
        if report is not None:
            report[0].copy_(report[1], non_blocking=True)
        return _record(self.main)

    def _drain(self, p, done, dst, src, out_host, per_slot=True):
        """dst := src, the output of the step of parity p whose event is `done`: host output on the D2H stream, one copy
        per slot (per_slot) or one, then out_copied[p]; device output on the main stream, one copy."""
        if not out_host:
            with torch.cuda.stream(self.main):
                dst.copy_(src, non_blocking=True)
            return
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(done)
            for d, s in zip(dst, src) if per_slot else ((dst, src),):
                d.copy_(s, non_blocking=True)
            self.out_copied[p] = _record(self.d2h)

    def _finish(self, cur, out_host, report=None):
        """End of a call: host output -> the report [k,...] (if any) copied to pinned host memory and one
        synchronisation; device output -> the current stream `cur` waits for the work of the call.  Returns the report
        as the caller reads it."""
        if out_host:
            if report is not None:       # the D2H stream has waited on the last replay's event
                k = report.shape[0]
                if self._report_host is None or self._report_host.shape[0] < k:
                    self._report_host = torch.empty(self._report_dev.shape, dtype=torch.int32, pin_memory=True)
                with torch.cuda.stream(self.d2h):
                    self.d2h.wait_stream(self.main)
                    self._report_host[:k].copy_(report, non_blocking=True)
                report = self._report_host[:k]
            self.d2h.synchronize()   # after every step (D2H waited on each) and so after every H2D
        else:
            cur.wait_stream(self.main)
            cur.wait_stream(self.h2d)    # a device input may be freed once the call returns
        return report


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
    'i444_10', or the 10-bit 4:2:2 'p210' / 'i422_10' / 'v210'): inp[p] holds [n,3h/2,w] frames ([n,h,2w] for 4:2:2,
    [n,3h,w] for 4:4:4, [n,2h,w] for P210 / I422_10, [n,h,v210_stride(w)] for v210; ops.yuv_word_dtype words) and
    the first launch is tg_stream_frame_in_yuv420 (8 bit, BT.601 limited range: cv2's conversion) or tg_stream_frame_in_yuv (any other layout or colour) instead, with the same reset.  YUV output
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

    Resized input (in_picture = (ph, pw)): the source picture is ph x pw and the net runs at h x w; the frame input is
    tg_stream_frame_in_resample instead, the same decode resized with the per-axis tables in_tables (rows, columns;
    built once) into lr[p] in the same one launch, with the same reset.  Everything after it sees the h x w frame:
    scene_cut scores the resized frames, and a padded stream's ring holds them.

    Windows (tg_frame_window).  crop = (Hf, Wf, top, left): inp[p] holds whole Hf x Wf source frames and the frame input
    reads the h x w picture at (top, left) out of them, in the same one launch (the net, FNet's flow and scene_cut see
    the picture only).  out_frame = (Hf, Wf, y, x): the copies out read padded frames, pad[p] (uint8 RGB [n,Hf,Wf,c])
    or yuv[p] (Hf x Wf YUV frames), whose bars are filled with the output format's black once, here, and never
    written again; every step writes the picture at (y, x) -- the windowed uint8 writer in place of the step's own
    uint8 output (the step then runs without it), the windowed resize, or the windowed encode.

    Copies overlap compute as in ClipEngine.run_clips.  uint8 input: inp[p] is itself the 2-deep staging ring (the
    step of parity p^1 never reads it), so the H2D of frame i+1 lands directly in the graph's input while frame i
    runs.  fp32 input: lr[p] is still read as lr_prev by frame i, so frames are staged as in run_clips."""

    def __init__(self, net, n, c, h, w, device, u8_input=True, bgr=False, yuv_in=None, yuv_out=None,
                 in_color='bt601', out_color='bt601', out_size=None, resize_filter='bicubic', scene_cut=None,
                 crop=None, out_frame=None, in_picture=None, in_filter='bicubic'):
        # lr / hr / u8 and the streams; the graphs are captured at the end, once the buffers below exist
        super().__init__(net, n, c, h, w, device, use_graph=False)
        dev, s = self.device, net.scale
        self.u8_input = u8_input or yuv_in is not None
        self.mask = [torch.zeros(n, dtype=torch.int32, device=dev) for _ in range(2)]
        self.crop = tuple(crop) if crop else None            # (Hf, Wf, top, left) of the input frames
        self.out_frame = tuple(out_frame) if out_frame else None   # (Hf, Wf, y, x) of the output frames
        self.in_picture = tuple(in_picture) if in_picture else None   # (ph, pw) of the source picture
        fh, fw = self.crop[:2] if self.crop else self.in_picture or (h, w)
        frame = ops.yuv_frame_shape(yuv_in, fh, fw) if yuv_in else (fh, fw, c)
        # 10-bit words: zeroed as int16, the same bits
        word = ops.yuv_word_dtype(yuv_in) if yuv_in else torch.uint8
        in_dtype = torch.int16 if word == torch.uint16 else torch.uint8
        self.inp = ([torch.zeros(n, *frame, dtype=in_dtype, device=dev).view(word) for _ in range(2)]
                    if self.u8_input else None)
        # the frame input, called as frame_in(frames, reset=, lr_curr=, lr_prev=, hr_prev=)
        in_window = self.crop[2:] if self.crop else None       # (top, left) of the picture in the input frames
        if in_window and yuv_in == 'v210':
            in_window = (*in_window, fw)                       # v210 rows do not give the frame's width: name it
        self.in_tables = None
        if self.in_picture:
            self.in_tables = [tuple(t.to(dev) for t in ops.resample_table(a, b, in_filter))
                              for a, b in zip(self.in_picture, (h, w))]
            self.frame_in = functools.partial(ops.stream_frame_in_resample, layout=yuv_in, color=in_color, scale=s,
                                              rows=self.in_tables[0], cols=self.in_tables[1], size=self.in_picture,
                                              bgr=bgr, window=in_window)
        elif yuv_in in YUV420 and in_color == 'bt601' and in_window is None:
            self.frame_in = functools.partial(ops.stream_frame_in_yuv420, layout=yuv_in, scale=s)
        elif yuv_in:
            # the windowed entry point has no BT.601-only twin: its bt601 row is the same cv2 conversion
            self.frame_in = functools.partial(ops.stream_frame_in_yuv, layout=yuv_in, color=in_color, scale=s,
                                              window=in_window)
        else:
            self.frame_in = functools.partial(ops.stream_frame_in, scale=s, bgr=bgr, window=in_window)
        # the output: per parity the step's own uint8 output step_u8[p] (or None), the calls after the step writes[p]
        # and the frames the copies out read res[p]
        H, W = self.H, self.W
        self.out_size = tuple(out_size) if out_size else None
        Ho, Wo = self.out_size or (H, W)
        out_window = self.out_frame[2:] if self.out_frame else None     # (y, x) of the picture in the output frames
        Yf, Xf = self.out_frame[:2] if self.out_frame else (Ho, Wo)
        enc_window = (*out_window, Xf) if out_window and yuv_out == 'v210' else out_window
        ten = yuv_out is not None and ops.yuv_depth(yuv_out) == 10
        self.yuv = self.pad = self.rs = self.tables = None
        if yuv_out:
            self.yuv = [torch.empty(n, *ops.yuv_frame_shape(yuv_out, Yf, Xf), dtype=ops.yuv_word_dtype(yuv_out),
                                    device=dev) for _ in range(2)]
        elif self.out_frame:
            self.pad = [torch.empty((n, Yf, Xf, c), dtype=torch.uint8, device=dev) for _ in range(2)]
        if self.out_frame:
            # on dev's current stream, which the capture's warm-up stream waits for: the fill is ordered before every
            # write of the picture
            with torch.cuda.device(dev):
                for t in self.yuv or self.pad:
                    if yuv_out == 'v210':
                        ops.fill_black_v210(t, out_color, Xf)
                    else:
                        ops.fill_black(t, yuv_out, out_color)
        if self.out_size:
            self.tables = [tuple(t.to(dev) for t in ops.resample_table(a, b, resize_filter))
                           for a, b in ((H, Ho), (W, Wo))]
            if not self.pad:      # uint8 [n,Ho,Wo,c], or fp32 [n,c,Ho,Wo] when a 10-bit encode follows
                self.rs = [torch.empty((n, c, Ho, Wo) if ten else (n, Ho, Wo, c),
                                       dtype=torch.float32 if ten else torch.uint8, device=dev) for _ in range(2)]
        src = self.rs or (self.hr if ten else self.u8)          # what an encode reads
        self.step_u8 = self.u8 if not self.out_size and not self.pad else [None, None]
        self.writes = [[], []]
        for p, calls in enumerate(self.writes):
            if self.out_size:
                dst = (dict(out_u8=self.pad[p], window=out_window) if self.pad else
                       {'out_f32' if ten else 'out_u8': self.rs[p]})
                calls.append(functools.partial(ops.resample, self.hr[p], *self.tables, **dst))
            elif self.pad:
                # the picture goes straight into the padded frame: the windowed writer replaces the step's uint8 output
                calls.append(functools.partial(ops.float_to_uint8_nhwc_window, self.hr[p], self.pad[p], out_window))
            if yuv_out in YUV420 and out_color == 'bt601' and out_window is None:
                calls.append(functools.partial(ops.rgb_u8_to_yuv420, src[p], yuv_out, out=self.yuv[p]))
            elif yuv_out:
                # 10 bit: from the step's fp32 HR frame (or its resize), two more bits than the uint8 output keeps
                calls.append(functools.partial(ops.rgb_to_yuv, yuv_out, out_color, out=self.yuv[p], window=enc_window,
                                               **{'rgb_f32' if ten else 'rgb_u8': src[p]}))
        self.res = self.yuv or self.pad or self.rs or self.u8
        self.scene_cut = scene_cut
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
        # the capture's warm-up steps update prev_mafd; that state is never read, because the first push resets every
        # slot (VideoStream._pending) and a reset sets prev_mafd := -1 without reading it
        self.use_graph = _use_graph()
        if self.use_graph:
            self._capture()

    def _enqueue(self, p):
        self.frame_in(self.inp[p] if self.inp else None, reset=self.mask[p], lr_curr=self.lr[p],
                      lr_prev=self.lr[p ^ 1], hr_prev=self.hr[p ^ 1])
        if self.scene_cut is not None:
            ops.scene_cut(self.lr[p], self.lr[p ^ 1], self.mask[p], self.scene_cut, self.prev_mafd, self.work,
                          self.score[p], self.cut[p])
            # a detected cut restarts the slot: the reset-only frame input with cut[p] as its mask
            ops.stream_frame_in(None, self.cut[p], self.lr[p], self.lr[p ^ 1], self.hr[p ^ 1], self.net.scale)
        self._step_out(p)

    def _step_out(self, p):
        """The step of parity p on lr[p], lr[p ^ 1], hr[p ^ 1] and the writes of its output frame."""
        self.net.step_into(self.lr[p], self.lr[p ^ 1], self.hr[p ^ 1], self.hr[p], out_u8=self.step_u8[p])
        for write in self.writes[p]:
            write()

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

    def _outputs(self, k, out_host):
        """The k frames a call returns (pinned host or device) and the [k,3n] report rows (scene_cut) or None."""
        n, res = self.n, self.res
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
        return out, report

    def run(self, frames, reset_slots, out_host, flush=False):
        """frames: uint8 [n,k,h,w,c] (u8_input), uint8 / uint16 [n,k,*yuv_frame_shape] (yuv_in) or fp32
        [n,k,c,h,w], each
        frame contiguous, pinned host or on this device; None for no frames.
        Slots in `reset_slots` start a new video at frame 0.  Returns uint8 [n,k,H,W,c] (or [n,k,3H/2,W] words with
        yuv_out; Ho, Wo instead of H, W with out_size): a pinned host tensor (out_host; one synchronisation, at the end) or a new tensor on the device,
        ordered on the current stream (no synchronisation).  flush: the videos end here (this engine holds no
        frames, so it changes nothing)."""
        k = 0 if frames is None else frames.shape[1]
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream()
            self.net.refresh_packed_weights()        # a load_state_dict between pushes takes effect
            for st in (self.main, self.h2d, self.d2h):
                st.wait_stream(cur)
            out, report = self._outputs(k, out_host)
            if not self.u8_input and self.stage is None:
                self.stage = [torch.empty_like(self.lr[0]) for _ in range(2)]
            dst = self.inp if self.u8_input else self.stage
            for i in range(k):
                p = self.parity
                staged = self._stage(dst[p], frames[:, i], self.in_free[p])
                with torch.cuda.stream(self.main):
                    self.main.wait_event(staged)
                    if not self.u8_input:
                        self.lr[p].copy_(self.stage[p], non_blocking=True)
                    self._set_mask(p, reset_slots if i == 0 else None)
                    copy = None if report is None else (report[i], self.rep[p])
                    self.in_free[p] = done = self._step(p, out_host, copy)
                self._drain(p, done, out[:, i], self.res[p], out_host)
                self.parity ^= 1
            self.report = self._finish(cur, out_host, report)
        return out


# ------------------------------------------------------------------------------------------ temporal padding
PAD_MODES = ('reflect', 'replicate')
MAX_PAD_FRONT = 32                # bounds the ring: pad_front + 2 decoded LR frames per slot
KEEP, ZERO, LOAD = ops.L.GATHER_KEEP, ops.L.GATHER_ZERO, ops.L.GATHER_LOAD


def pad_count(p, mode, length):
    """Pad frames in front of a shot of `length` frames: reflect min(p, length - 1) (the reference asserts
    p < length; the stream pads with the longest reflection the shot has), replicate p."""
    return min(p, length - 1) if mode == 'reflect' else p


def shot_lengths(j, starts, end, p):
    """Per slot: None when frame j continues a shot, else the length of the shot that starts at j, capped at p + 1.
    starts: per slot the set of frames that start a shot, known up to j + p; end: the frame count when the videos
    end before j + p + 1 (a flush), else None."""
    out = []
    for b in starts:
        if j not in b:
            out.append(None)
            continue
        length = p + 1
        for i in range(1, p + 1):
            if j + i in b or (end is not None and j + i >= end):
                length = i
                break
        out.append(length)
    return out


def plan_step(j, lengths, p, mode):
    """The warm-up steps and the main step that produce lock-stepped frame j of a stream padded as
    BaseModel.pad_sequence pads each shot (base_model.py:230-251).  lengths: shot_lengths(j, ...).
    -> (warm, main):
      warm: the warm-up steps in order, each a per-slot list of (cur, mode): cur the frame read as lr_curr (None:
            nothing is read), mode ZERO at the slot's first warm-up step (zero state, as frame 0 of infer_sequence),
            else KEEP.  A shot with q pad frames runs q steps over its pad frames (reflect: j+q, ..., j+1; replicate:
            j, ..., j), ending on the last step of the list: slots that start a shot at j share the steps.
      main: per slot (j, mode, prev): KEEP continues the shot; ZERO starts it cold (no pad frame); LOAD starts it from
            the warm-up: hr_prev is the warm-up's last HR frame and lr_prev is frame prev (its last pad frame)."""
    qs = [None if length is None else pad_count(p, mode, length) for length in lengths]
    qmax = max([q for q in qs if q] or [0])
    warm = [[(None, KEEP)] * len(qs) for _ in range(qmax)]
    main = []
    for k, q in enumerate(qs):
        if q is None:
            main.append((j, KEEP, None))
        elif q == 0:
            main.append((j, ZERO, None))
        else:
            for m in range(q):
                warm[qmax - q + m][k] = (j + q - m if mode == 'reflect' else j, ZERO if m == 0 else KEEP)
            main.append((j, LOAD, j + 1 if mode == 'reflect' else j))
    return warm, main


def plan(starts, frames, p, mode):
    """The whole schedule of `frames` lock-stepped frames whose shots start at `starts` (per slot, a set of frames;
    frame 0 starts every slot's first shot) and end with the stream: [plan_step(j, ...) for j in range(frames)]."""
    starts = [set(b) | {0} for b in starts]
    return [plan_step(j, shot_lengths(j, starts, frames, p), p, mode) for j in range(frames)]


class PadSchedule:
    """The host's plan of a padded stream of n lock-stepped slots: the shot starts seen so far, the next frame to
    ingest (t_in) and to produce (t_out).  Pure Python; PaddedStreamEngine calls, per push: start(reset slots), then
    per frame ingest(cut slots) and next() while ready(); per flush: next(flush=True) while ready(flush=True), then
    restart()."""

    def __init__(self, n, p, mode):
        self.n, self.p, self.mode = n, p, mode
        self.lag = p if mode == 'reflect' else 0
        self.t_in = self.t_out = 0
        self.starts = [set() for _ in range(n)]      # per slot, the frames not yet produced that start a shot

    def start(self, slots):
        """`slots` start a new video at the next frame ingested (the caller's resets)."""
        for k in slots:
            self.starts[k].add(self.t_in)

    def ingest(self, cut_slots=()):
        """Frame t_in is in the ring; `cut_slots` detected a scene cut at it."""
        self.start(cut_slots)
        self.t_in += 1

    def ready(self, flush=False):
        """Frame t_out can be produced: frames up to t_out + lag are ingested, or the videos end (flush)."""
        return self.t_out < self.t_in - (0 if flush else self.lag)

    def next(self, flush=False):
        """-> (j, warm, main) of frame j = t_out (plan_step), which the caller then produces."""
        j = self.t_out
        warm, main = plan_step(j, shot_lengths(j, self.starts, self.t_in if flush else None, self.p), self.p,
                               self.mode)
        self.t_out += 1
        for b in self.starts:                          # frames before t_out never start a planned shot again
            b.discard(j)
        return j, warm, main

    def restart(self):
        """After a flush: every slot starts a new video at the next frame."""
        assert self.t_out == self.t_in
        self.start(range(self.n))


class PaddedStreamEngine(StreamEngine):
    """StreamEngine for a stream padded at every shot start (FRNet.stream(pad_front=p)).

    Ingest: each pushed frame t is decoded (the frame-input launch, no reset) into ring[t % depth], a device ring of
    depth = p + 2 fp32 LR frames [depth,n,c,h,w], and with scene_cut scored against ring[(t-1) % depth] on the ingest
    stream; the cut flags go to pinned host memory, and the host reads them from there.  The caller's resets and
    the cuts are the shot starts of each slot.

    Frame j is produced once frames up to j + lag (lag = p for 'reflect', 0 for 'replicate') are ingested, or the
    videos end (flush): plan_step gives its warm-up steps -- batch-n graphs on their own state wlr / whr, each starting
    with tg_stream_gather of the table wtab[q] -- and its main step, the main graph of parity p: tg_stream_gather of
    mtab[p] (lr[p] = ring[j % depth]; per slot keep, zero, or load lr_prev from the ring and hr_prev from whr[0]), the
    unchanged net.step_into and the output writes of StreamEngine.  The tables are int32 [3n] in device memory,
    written by one H2D copy before each replay, so the four captured graphs serve every schedule."""

    def __init__(self, net, n, c, h, w, device, pad_front, padding_mode, **kw):
        dev = torch.device(device)
        self.sched = PadSchedule(n, pad_front, padding_mode)
        self.depth = pad_front + 2
        H, W = net.scale * h, net.scale * w
        self.ring = torch.zeros((self.depth, n, c, h, w), device=dev)
        self.wlr = [torch.zeros(n, c, h, w, device=dev) for _ in range(2)]
        self.whr = [torch.zeros(n, c, H, W, device=dev) for _ in range(2)]
        idle = torch.tensor([-1] * n + [KEEP] * n + [-1] * n, dtype=torch.int32)
        self.mtab = [idle.to(dev) for _ in range(2)]
        self.wtab = [idle.to(dev) for _ in range(2)]
        self.warm_graphs = [None, None]
        self.ingest = torch.cuda.Stream(device=dev)
        self.ring_free = [None] * self.depth         # event: the main step that last read ring[r] finished
        self.ingested = None                         # event: the latest ingest finished
        self.rep_ring = self.cut_host = self.in_mask = None
        if kw.get('scene_cut') is not None:
            # per ring position the frame's report: [0,2n) the float64 scores, [2n,3n) the cut flags; rows of 4n words
            # keep every row's scores 8-byte aligned
            self.rep_ring = torch.zeros((self.depth, 4 * n), dtype=torch.int32, device=dev)
            self.cut_host = torch.zeros((self.depth, n), dtype=torch.int32, pin_memory=True)
            self.in_mask = torch.zeros(n, dtype=torch.int32, device=dev)
        super().__init__(net, n, c, h, w, dev, **kw)

    def _enqueue(self, p):
        ops.stream_gather(self.ring, self.mtab[p], self.whr[0], self.lr[p], self.lr[p ^ 1], self.hr[p ^ 1],
                          self.net.scale)
        self._step_out(p)

    def _enqueue_warm(self, q):
        ops.stream_gather(self.ring, self.wtab[q], None, self.wlr[q], self.wlr[q ^ 1], self.whr[q ^ 1], self.net.scale)
        self.net.step_into(self.wlr[q], self.wlr[q ^ 1], self.whr[q ^ 1], self.whr[q], out_u8=None)

    def _capture(self):
        super()._capture()
        with torch.cuda.device(self.device):
            warm = torch.cuda.Stream(device=self.device)
            warm.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(warm):
                for q in (0, 1):
                    self._enqueue_warm(q)
            torch.cuda.current_stream().wait_stream(warm)
            torch.cuda.synchronize(self.device)
            for q in (0, 1):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, pool=self.graphs[1].pool()):
                    self._enqueue_warm(q)
                self.warm_graphs[q] = g

    def run_warm(self, q):
        if self.warm_graphs[q] is not None:
            self.warm_graphs[q].replay()
        else:
            self._enqueue_warm(q)

    def _load_table(self, tab, rows):
        """On the current stream: tab = cur + mode + prev of rows [(cur, mode, prev)] (frames -> ring positions)."""
        pos = lambda f: -1 if f is None else f % self.depth          # noqa: E731
        vals = [pos(r[0]) for r in rows] + [r[1] for r in rows] + [pos(r[2] if len(r) > 2 else None) for r in rows]
        tab.copy_(torch.tensor(vals, dtype=torch.int32).pin_memory(), non_blocking=True)

    def run(self, frames, reset_slots, out_host, flush=False):
        """StreamEngine.run with padding: returns the frames that are complete after this call's frames are ingested,
        [n,k_out,...], k_out = the frames up to lag behind the last ingested one (flush: all of them); the report
        rows (scene_cut) are those of the returned frames."""
        sched, k = self.sched, 0 if frames is None else frames.shape[1]
        end = sched.t_in + k
        k_out = max(0, (end if flush else end - sched.lag) - sched.t_out)
        with torch.cuda.device(self.device):
            cur = torch.cuda.current_stream()
            self.net.refresh_packed_weights()
            for st in (self.main, self.h2d, self.d2h, self.ingest):
                st.wait_stream(cur)
            out, report = self._outputs(k_out, out_host)
            sched.start(reset_slots)
            row = 0
            for i in range(k):
                self._ingest(frames, i, reset_slots if i == 0 else ())
                while sched.ready():
                    self._emit(row, out, report, out_host, *sched.next())
                    row += 1
            while flush and sched.ready(flush=True):
                self._emit(row, out, report, out_host, *sched.next(flush=True))
                row += 1
            if flush:
                sched.restart()
            assert row == k_out
            if out_host:
                self.ingest.synchronize()              # the H2D of the frames held for later steps too
            else:
                cur.wait_stream(self.ingest)
            self.report = self._finish(cur, out_host, report)
        return out

    def _ingest(self, frames, i, reset_slots):
        t, n = self.sched.t_in, self.n
        r = t % self.depth
        q = t & 1                                      # staging buffer of uint8 / YUV input
        if self.u8_input:
            staged = self._stage(self.inp[q], frames[:, i], self.in_free[q])
        else:                                          # fp32 frames land in the ring directly
            staged = self._stage(self.ring[r], frames[:, i], self.ring_free[r])
        with torch.cuda.stream(self.ingest):
            self.ingest.wait_event(staged)
            _wait(self.ingest, self.ring_free[r])
            if self.u8_input:
                # no reset: lr_prev / hr_prev are not touched
                self.frame_in(self.inp[q], reset=None, lr_curr=self.ring[r], lr_prev=self.lr[0], hr_prev=self.hr[0])
                self.in_free[q] = _record(self.ingest)
            if self.scene_cut is not None:
                mask = None
                if reset_slots:
                    m = torch.zeros(n, dtype=torch.int32)
                    m[list(reset_slots)] = 1
                    self.in_mask.copy_(m.pin_memory(), non_blocking=True)
                    mask = self.in_mask
                rep = self.rep_ring[r]
                ops.scene_cut(self.ring[r], self.ring[(t - 1) % self.depth], mask, self.scene_cut, self.prev_mafd,
                              self.work, rep[:2 * n].view(torch.float64), rep[2 * n:3 * n])
                self.cut_host[r].copy_(rep[2 * n:3 * n], non_blocking=True)
            self.ingested = _record(self.ingest)
        cuts = ()
        if self.scene_cut is not None:
            self.ingested.synchronize()                # the ingest only: decode, score and the flag copy
            cuts = [int(k) for k in np.flatnonzero(self.cut_host[r].numpy())]
        self.sched.ingest(cuts)

    def _emit(self, row, out, report, out_host, j, warm, main):
        """Warm-ups and main step of frame j, its output into out[:, row] and its report into report[row]."""
        r = j % self.depth
        with torch.cuda.stream(self.main):
            self.main.wait_event(self.ingested)       # frames up to t_in - 1 are in the ring
            for i, step in enumerate(warm):
                q = (len(warm) - 1 - i) & 1             # the last warm-up writes whr[0], which the main step loads
                self._load_table(self.wtab[q], step)
                self.run_warm(q)
            p = self.parity
            self._load_table(self.mtab[p], main)
            copy = None if report is None else (report[row], self.rep_ring[r, :3 * self.n])
            self.ring_free[r] = done = self._step(p, out_host, copy)
        self._drain(p, done, out[:, row], self.res[p], out_host)
        self.parity ^= 1


YUV420 = ops.YUV420_LAYOUTS       # 'nv12', 'i420'
YUV = ops.YUV_LAYOUTS             # those, the 10-bit 'p010', 'i420_10', 4:2:2 'yuy2', 'uyvy', 4:4:4 'i444', 'i444_10',
                                  # 10-bit 4:2:2 'p210', 'i422_10', 'v210'
COLORS = ops.YUV_COLORS           # 'bt601' (the default, cv2's conversion), 'bt709', 'bt601-full', 'bt709-full'


class VideoStream:
    """n lock-stepped video slots through FRNet with the recurrent state carried between `push` calls.
    Created by FRNet.stream(); see there."""

    def __init__(self, net, n, h, w, device=None, input='uint8', channel_order='rgb', out_format='rgb',
                 in_color='bt601', out_color='bt601', out_size=None, resize_filter='bicubic', scene_cut=None,
                 crop=None, out_frame=None, out_origin=None, pad_front=0, padding_mode='reflect', in_size=None,
                 in_filter='bicubic'):
        if not _is_int(pad_front) or not 0 <= pad_front <= MAX_PAD_FRONT:
            raise ValueError(f'pad_front must be an int in [0, {MAX_PAD_FRONT}], got {pad_front!r}')
        if not isinstance(padding_mode, str) or padding_mode not in PAD_MODES:
            raise ValueError(f'padding_mode must be one of {PAD_MODES}, got {padding_mode!r}')
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
        if not isinstance(in_filter, str) or in_filter not in ops.RESIZE_FILTERS:
            raise ValueError(f'in_filter must be one of {ops.RESIZE_FILTERS}, got {in_filter!r}')
        if in_size is None and in_filter != 'bicubic':
            raise ValueError(f'in_filter={in_filter!r} applies to a resized input only (give in_size)')
        if in_size is not None and input == 'float32':
            raise ValueError("in_size applies to uint8 and YUV frames, not to input='float32'")
        if crop is not None:
            if input == 'float32':
                raise ValueError("crop applies to uint8 and YUV frames, not to input='float32'")
            crop = _check_box('crop', crop, h, w, input)
        ph, pw = crop[2:] if crop else (h, w)      # the source picture
        if in_size is not None:
            in_size = _check_in_size(in_size, ph, pw)
        ph, pw = in_size or (ph, pw)               # the picture the net runs on
        if out_size is not None:
            out_size = _check_out_size(out_size, net.scale * ph, net.scale * pw, out_format)
        yuv = [f for f in (input, out_format) if f in YUV]
        # the input layout holds the pushed h x w frames; the output layout's picture comes from the ph x pw picture
        # the net runs on (the whole frame without crop)
        for f, (a, b) in ((input, (h, w)), (out_format, (ph, pw))):
            err = f in YUV and ops.yuv_size_error(f, a, b)
            if err:
                raise ValueError(f'{f} frames: {err}')
        if out_frame is None and out_origin is not None:
            raise ValueError('out_origin applies to a padded output only (give out_frame)')
        if out_frame is not None:
            Ho, Wo = out_size or (net.scale * ph, net.scale * pw)
            out_frame, out_origin = _check_out_frame(out_frame, out_origin, Ho, Wo, out_format)
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
        self.crop, self.out_frame, self.out_origin = crop, out_frame, out_origin
        self.pad_front, self.padding_mode = int(pad_front), padding_mode
        self.in_size, self.in_filter = in_size, in_filter
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
        'i444_10' uint16 [n,k,3h,w] (H, W or Ho, Wo on the output side).  10-bit 4:2:2: 'p210' / 'i422_10' uint16
        [n,k,2h,w] and 'v210' uint8 [n,k,h,S] with S = 128 * ceil(w / 48) bytes a row.
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
        return self._result(res, out)

    def flush(self, out='host'):
        """End every slot's video: returns the frames the stream still holds, [n,k_held,...] as push returns them
        (k_held <= pad_front with padding_mode='reflect', 0 otherwise), each made with the padding its shot gets
        now that the shot's end is known; last_cuts / last_scores describe them.  Every slot then starts a new video
        at the next push, as in a new stream."""
        if self._engine is False:
            raise ops.L.TecoganB200Error('VideoStream.flush: the stream is closed')
        if out not in ('host', 'device'):
            raise ValueError(f"out must be 'host' or 'device', got {out!r}")
        _check_inference(self.net)
        if self._engine is None:
            self._engine = self._build()
        res = self._engine.run(None, [], out == 'host', flush=True)
        self._pending = [True] * self.n
        return self._result(res, out)

    def _result(self, res, out):
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
        dtype = (torch.float32 if self.input == 'float32' else
                 ops.yuv_word_dtype(self.input) if self.input in YUV else torch.uint8)
        if frames.dtype != dtype:
            raise L.TecoganB200Error(f'VideoStream.push: {self.input} stream expects {dtype} frames, got '
                                     f'{frames.dtype}')
        frame, layout = {'uint8': ((self.h, self.w, self.c), 'n,k,h,w,c'),
                         'float32': ((self.c, self.h, self.w), 'n,k,c,h,w')}.get(
                             self.input, (None, None))
        if frame is None:
            frame = ops.yuv_frame_shape(self.input, self.h, self.w)
            layout = 'n,k,' + ops.YUV_LAYOUT_TABLE[self.input].text
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
        engine, args, kw = self._engine_args()
        return engine(*args, **kw)

    def _engine_args(self):
        """(engine class, positional arguments, keyword arguments) of the stream's engine."""
        yuv_in = self.input if self.input in YUV else None
        yuv_out = self.out_format if self.out_format in YUV else None
        h, w, crop = self.h, self.w, None
        if self.crop:
            top, left, h, w = self.crop
            crop = (self.h, self.w, top, left)
        out_frame = (*self.out_frame, *self.out_origin) if self.out_frame else None
        engine, kw = StreamEngine, {}
        if self.pad_front:
            engine, kw = PaddedStreamEngine, dict(pad_front=self.pad_front, padding_mode=self.padding_mode)
        if self.in_size is not None and self.in_size != (h, w):
            # the net runs at in_size; an in_size equal to the picture is the stream without it
            kw.update(in_picture=(h, w), in_filter=self.in_filter)
            h, w = self.in_size
        return engine, (self.net, self.n, self.c, h, w, self.device), dict(
            u8_input=self.input == 'uint8', bgr=self.channel_order == 'bgr', yuv_in=yuv_in, yuv_out=yuv_out,
            in_color=self.in_color, out_color=self.out_color, out_size=self.out_size,
            resize_filter=self.resize_filter, scene_cut=self.scene_cut, crop=crop, out_frame=out_frame, **kw)


def _check_scene_cut(threshold):
    """scene_cut -> float threshold, or ValueError: a real number (not a bool) in (0, 100]; NaN and inf refused."""
    if isinstance(threshold, bool) or not isinstance(threshold, numbers.Real):
        raise ValueError(f'scene_cut must be None or a threshold in (0, 100], got {threshold!r}')
    t = float(threshold)
    if not (math.isfinite(t) and ops.scene_cut_threshold_ok(t)):
        raise ValueError(f'scene_cut threshold must be finite and in (0, 100], got {threshold!r}')
    return t


def _check_in_size(in_size, h, w):
    """in_size -> (hn, wn) ints, or ValueError: two positive ints within the resize's ratios (1/4 to 2 times) of the
    h x w source picture."""
    if (not isinstance(in_size, (tuple, list)) or len(in_size) != 2
            or not all(_is_int(v) and v > 0 for v in in_size)):
        raise ValueError(f'in_size must be (hn, wn), two positive ints, got {in_size!r}')
    hn, wn = int(in_size[0]), int(in_size[1])
    if not (ops.resample_ratio_ok(h, hn) and ops.resample_ratio_ok(w, wn)):
        raise ValueError(f'in_size {hn}x{wn} from a {h}x{w} picture: each axis must be within 1/4 to 2 times the '
                         f'picture size')
    return hn, wn


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
    err = out_format in YUV and ops.yuv_size_error(out_format, Ho, Wo)
    if err:
        raise ValueError(f'{out_format} frames: out_size {Ho}x{Wo}: {err}')
    return Ho, Wo


def _is_int(v):
    return isinstance(v, numbers.Integral) and not isinstance(v, bool)


def _grids(layout):
    """(row, column) steps of a layout's chroma grid, where a picture starts (4:2:0 (2, 2), 4:2:2 (1, 2), RGB / 4:4:4
    (1, 1); v210 (1, 6), its 6-pixel groups), and of its frame and picture sizes (the same, except v210's even width:
    a picture that reaches the frame's right edge may end inside a group)."""
    if layout not in YUV:
        return (1, 1), (1, 1)
    lay = ops.YUV_LAYOUT_TABLE[layout]
    return lay.grid, lay.size_grid


def _group_end(layout, right, w):
    """A picture ending at column `right` of a w-wide frame ends on the layout's grid: always, except in v210, whose
    pictures end on a 6-pixel group or at the frame's right edge."""
    return layout != 'v210' or right % 6 == 0 or right == w


def _check_box(arg, box, h, w, layout):
    """box = (top, left, ch, cw) -> ints, or ValueError: a non-empty box inside the h x w frame, on the layout's
    chroma grid (4:2:0: all four even; 4:2:2: left and cw even; v210: left on a 6-pixel group, cw even and the box
    ending on a group or at the frame's right edge)."""
    if not isinstance(box, (tuple, list)) or len(box) != 4 or not all(_is_int(v) for v in box):
        raise ValueError(f'{arg} must be (top, left, ch, cw), four ints, got {box!r}')
    top, left, ch, cw = (int(v) for v in box)
    if top < 0 or left < 0 or ch <= 0 or cw <= 0 or top + ch > h or left + cw > w:
        raise ValueError(f'{arg} {ch}x{cw} at ({top}, {left}) lies outside the {h}x{w} frame')
    (gy, gx), (sy, sx) = _grids(layout)
    if top % gy or ch % sy or left % gx or cw % sx or not _group_end(layout, left + cw, w):
        raise ValueError(f'{arg} ({top}, {left}, {ch}, {cw}) is off the {layout} chroma grid: rows in steps of {gy}, '
                         f'columns in steps of {gx}' + _V210_RULE * (layout == 'v210'))
    return top, left, ch, cw


_V210_RULE = ' (a v210 picture starts on a 6-pixel group and ends on one or at the frame\'s right edge)'


def _check_out_frame(out_frame, out_origin, Ho, Wo, out_format):
    """out_frame (Hf, Wf) and out_origin (y, x) or None -> ints, or ValueError: the Ho x Wo picture inside the frame,
    frame and origin on the output layout's chroma grid.  The default origin centres the picture, rounded down to
    the grid; a v210 picture that would then not end on a 6-pixel group goes to the frame's right edge instead, the
    only place it can end inside a group."""
    if (not isinstance(out_frame, (tuple, list)) or len(out_frame) != 2
            or not all(_is_int(v) and v > 0 for v in out_frame)):
        raise ValueError(f'out_frame must be (Hf, Wf), two positive ints, got {out_frame!r}')
    Hf, Wf = int(out_frame[0]), int(out_frame[1])
    if Ho > Hf or Wo > Wf:
        raise ValueError(f'the {Ho}x{Wo} output picture does not fit out_frame {Hf}x{Wf}')
    (gy, gx), (sy, sx) = _grids(out_format)
    if Hf % sy or Wf % sx:
        raise ValueError(f'out_frame {Hf}x{Wf} is off the {out_format} chroma grid')
    if out_origin is None:
        x = (Wf - Wo) // 2 // gx * gx
        if not _group_end(out_format, x + Wo, Wf):
            if (Wf - Wo) % gx:
                raise ValueError(f'no out_origin puts a {Wo}-wide v210 picture into out_frame {Hf}x{Wf}: it starts on '
                                 f'a 6-pixel group and ends on one or at the frame\'s right edge, so Wo or Wf - Wo '
                                 f'must be a multiple of 6')
            x = Wf - Wo
        out_origin = ((Hf - Ho) // 2 // gy * gy, x)
    if not isinstance(out_origin, (tuple, list)) or len(out_origin) != 2 or not all(_is_int(v) for v in out_origin):
        raise ValueError(f'out_origin must be (y, x), two ints, got {out_origin!r}')
    y, x = int(out_origin[0]), int(out_origin[1])
    if y < 0 or x < 0 or y + Ho > Hf or x + Wo > Wf:
        raise ValueError(f'the {Ho}x{Wo} output picture at out_origin ({y}, {x}) does not fit out_frame {Hf}x{Wf}')
    if y % gy or x % gx or not _group_end(out_format, x + Wo, Wf):
        raise ValueError(f'out_origin ({y}, {x}) is off the {out_format} chroma grid' +
                         _V210_RULE * (out_format == 'v210'))
    return (Hf, Wf), (y, x)


def fit_size(picture, frame, sar=(1, 1), out_format='rgb'):
    """The largest picture size (h, w) that shows a `picture` (ch, cw) of sample aspect ratio `sar` at its display
    aspect inside `frame` (Hf, Wf) of square pixels: letterboxed or pillarboxed, each side on out_format's chroma grid
    and within the resize's ratios (1/4 to 2 times the picture's side).  Host only.  Use it as out_size with
    out_frame=frame: an anamorphic 720x480 DVD (sar 8:9 for 4:3, 32:27 for 16:9) becomes a pillarbox or letterbox of
    a 1080p frame.  The ratio limits refer to the picture given here; pass the HR size (scale * crop) as `picture`
    for a stream.  ValueError when no size on the grid fits."""
    for arg, v in (('picture', picture), ('frame', frame), ('sar', sar)):
        if not isinstance(v, (tuple, list)) or len(v) != 2 or not all(_is_int(x) and x > 0 for x in v):
            raise ValueError(f'{arg} must be two positive ints, got {v!r}')
    if out_format not in ('rgb', *YUV):
        raise ValueError(f"out_format must be 'rgb' or one of {YUV}, got {out_format!r}")
    ch, cw = (int(v) for v in picture)
    Hf, Wf = (int(v) for v in frame)
    gy, gx = _grids(out_format)[0]
    # display aspect num / den = (cw * sar_w) / (ch * sar_h), exact in integers
    num, den = cw * int(sar[0]), ch * int(sar[1])
    h, w = Hf, Hf * num // den
    if w > Wf:
        w, h = Wf, Wf * den // num
    h, w = min(h // gy * gy, 2 * ch // gy * gy), min(w // gx * gx, 2 * cw // gx * gx)
    # the side the ratio capped first keeps the display aspect of the other (rounded down to the grid)
    if h * num > w * den:
        h = w * den // num // gy * gy
    elif w * den > h * num:
        w = h * num // den // gx * gx
    if h <= 0 or w <= 0 or not (ops.resample_ratio_ok(ch, h) and ops.resample_ratio_ok(cw, w)):
        raise ValueError(f'no {out_format} picture size between 1/4 and 2 times {ch}x{cw} fits {Hf}x{Wf} at aspect '
                         f'{num}:{den}')
    return h, w


def detect_bars(frames, input='uint8', channel_order='rgb', limit=24, width=None):
    """The picture box (top, left, ch, cw) of letterboxed / pillarboxed frames, found on the device: a row or column
    is picture when its mean 8-bit luma exceeds `limit` in any of the frames (24 is ffmpeg cropdetect's default
    limit; the rule is oracle/frame_window.py's, not cropdetect's), and the box spans the first to the last picture
    row and column, rounded inward to the input layout's chroma grid.  Luma is Y for YUV input (10-bit samples >> 2)
    and cv2's gray of RGB ((9798 R + 19235 G + 3735 B + 16384) >> 15).  frames: a CUDA tensor [k,h,w,3] (uint8,
    channel_order 'rgb' or 'bgr') or [k,*yuv_frame_shape(input, h, w)] for a YUV input.  Frames with no picture row
    or column (all black) give the whole frame.  v210 frames [k,h,128*ceil(w/48)] need their width w (`width`), which
    their padded rows do not give; their box starts on a 6-pixel group and ends on one or at the frame's right edge.
    Pass crop=detect_bars(...) to FRNet.stream."""
    if input not in ('uint8', *YUV):
        raise ValueError(f"input must be 'uint8' or one of {YUV}, got {input!r}")
    if channel_order not in ('rgb', 'bgr') or (input != 'uint8' and channel_order != 'rgb'):
        raise ValueError(f'channel_order={channel_order!r} does not apply to input={input!r}')
    if isinstance(limit, bool) or not isinstance(limit, numbers.Real) or not 0 <= limit < 255:
        raise ValueError(f'limit must be a number in [0, 255), got {limit!r}')
    if (width is None) != (input != 'v210'):
        raise ValueError(f'width applies to, and is needed by, v210 frames only (input={input!r}, width={width!r})')
    if not isinstance(frames, torch.Tensor) or not frames.is_cuda:
        raise ValueError('detect_bars: frames must be a CUDA tensor')
    layout = input if input in YUV else None
    with torch.cuda.device(frames.device):          # the memsets and the kernel go to the frames' device
        rows, cols = ops.luma_line_sums(frames.contiguous(), layout, channel_order == 'bgr', frame_w=width)
    h, w = rows.shape[1], cols.shape[1]
    # mean > limit <=> sum > limit * count: exact for integer limits, and for others compared in float64
    pic_r = (rows.double() > float(limit) * w).any(0).cpu().numpy()
    pic_c = (cols.double() > float(limit) * h).any(0).cpu().numpy()
    return bars_box(pic_r, pic_c, input)


def bars_box(pic_rows, pic_cols, layout):
    """(top, left, ch, cw) from per-row / per-column picture flags, rounded inward to the layout's chroma grid; the
    whole frame when no row or column is picture (or the rounded box is empty)."""
    h, w = len(pic_rows), len(pic_cols)
    gy, gx = _grids(layout)[0]
    if not pic_rows.any() or not pic_cols.any():
        return 0, 0, h, w
    r = np.flatnonzero(pic_rows)
    c = np.flatnonzero(pic_cols)
    top, bottom = -(-int(r[0]) // gy) * gy, (int(r[-1]) + 1) // gy * gy
    left, right = -(-int(c[0]) // gx) * gx, (int(c[-1]) + 1) // gx * gx
    if layout == 'v210' and int(c[-1]) + 1 == w:
        right = w                                    # a v210 picture may end inside the frame's last group
    if bottom <= top or right <= left:
        return 0, 0, h, w
    return top, left, bottom - top, right - left


def _check_inference(net):
    if net.training and any(p.requires_grad for p in net.parameters()):
        raise ops.L.TecoganB200Error('FRNet.stream is inference only: call net.eval() (or set requires_grad=False '
                                     'on the parameters) first')
