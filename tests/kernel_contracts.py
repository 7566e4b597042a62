"""TEST INFRASTRUCTURE ONLY -- replays every op call of a training step or of an inference step against its
contract in tests/fake_ops.py, on the arguments the step actually passes.

A Recorder wraps, on the package's op layer, exactly the names fake_ops.install replaces (the PackedConv /
PackedDgrad / GradScale classes through subclasses that also note each layer's fp32 weight and bias).  For
every top-level call it

  * copies every tensor argument to the CPU before the call (in-place outputs too: dw, db, d_hr_prev, y of an
    accumulating upsample), and poisons write-only outputs with NaN (uint8 ones with the byte 77);
  * runs the stand-in on those copies in float64 (weights rounded to fp16 as the kernels store them), so each
    call is judged on its own inputs and errors do not compound;
  * compares every output per element: data movement and the loss scale bit for bit; arithmetic against
    |got - ref| <= ulp_out(ref) + gamma_K * (the same op on |operands|), gamma_K = K u / (1 - K u), u = 2^-24,
    K the number of addends (plus a coordinate-rounding term for the bilinear warps).  ulp_out(0) = 0: pad
    channels and poisoned buffers must come back exactly written.

Ops with a bound of their own: a pooled conv is held to the max-pool of its unpooled bound; fused_tail's fp32 frame
to a bound that carries the fp16 HR map through conv_out (Recorder._tail), and its uint8 frame to the bits of
float32_to_uint8 of that fp32 frame.

Launches through the op layer from outside a wrapped call are collected as `unfaked`, so a kernel that enters
the training or inference path without a stand-in is reported.
"""
import inspect
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, 'tests')):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import fake_ops as FK                         # noqa: E402

U = 2.0 ** -24
F64 = torch.float64

# op -> arguments it writes.  Write-only outputs (not read by the op) are poisoned before the call.
OUTPUTS = {
    'PackedConv': ('y',), 'PackedDgrad': ('y',), 'wgrad': ('dw', 'db'), 'bias_grad': ('db',), 'grad_pack': ('y',),
    'pack_pair': ('y',), 'nchw_to_nhwc': ('y',), 'maxpool2x2': ('y',), 'upsample2x': ('y',), 'upsample': ('y',),
    'upsample_bwd': ('gx',), 'warp_s2d_concat_hrflow': ('out',), 'warp_s2d_concat_bwd': ('d_hr_prev', 'd_hr_flow'),
    'maxpool2x2_bwd': ('gx',), 'upsample2x_bwd': ('gx',), 'flow_head_bwd': ('dz',), 'backward_warp': ('y',),
    'backward_warp_bwd': (), 'space_to_depth': ('y',), 'depth_to_space': (), 'GradScale': (),
    'fused_tail': ('y', 'y_u8'), 'warp_s2d_concat_lrflow': ('out',), 'float_to_uint8_nhwc': ('y',),
}
ACCUMULATING = {('wgrad', 'dw'), ('wgrad', 'db'), ('bias_grad', 'db'), ('warp_s2d_concat_bwd', 'd_hr_prev')}
EXACT = {'pack_pair', 'nchw_to_nhwc', 'space_to_depth', 'depth_to_space', 'grad_pack', 'maxpool2x2', 'GradScale',
         'float_to_uint8_nhwc'}
WARPS = {'warp_s2d_concat_hrflow', 'warp_s2d_concat_lrflow', 'warp_s2d_concat_bwd', 'backward_warp', 'backward_warp_bwd'}


def gamma(k):
    return k * U / (1 - k * U)


def ulp(ref, dtype):
    """spacing of `dtype` at |ref| (float64 tensor); 0 where ref == 0"""
    emin, p = (-14, 10) if dtype == torch.float16 else (-126, 23)
    a = ref.abs()
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** emin)))
    return torch.where(a == 0, torch.zeros_like(a), torch.exp2(e - p))


class _Mode:
    """fake_ops computing in float64 without rounding (optionally with |filter taps|)"""

    def __init__(self, absolute=False):
        self.absolute = absolute

    def __enter__(self):
        self.saved = FK.STORAGE, FK.COMPUTE, FK.ABS_TAPS
        FK.STORAGE = FK.COMPUTE = F64
        FK.ABS_TAPS = self.absolute

    def __exit__(self, *exc):
        FK.STORAGE, FK.COMPUTE, FK.ABS_TAPS = self.saved


def _overlaps(a, b):
    if a.device != b.device:
        return False
    a0, b0 = a.data_ptr(), b.data_ptr()
    return a0 < b0 + b.numel() * b.element_size() and b0 < a0 + a.numel() * a.element_size()


def _poison(t):
    t.fill_(77 if t.dtype == torch.uint8 else float('nan'))     # uint8 holds no NaN: a fixed byte instead


class Recorder:
    def __init__(self, ops, monkeypatch, names=FK.FAKED):
        self.ops = ops
        self.depth = 0
        self.params = {}            # id(layer object) -> (fp32 weight, fp32 bias or None) on the CPU
        self.layers = {}            # id(layer object) -> the object (kept alive)
        self.seen = set()
        self.calls = {}             # op -> number of checked calls
        self.worst = {}             # op -> worst |err| / bound
        self.failures = []
        self.unfaked = []
        for name in names:
            real = getattr(ops, name)
            wrapped = self._wrap_class(name, real) if inspect.isclass(real) else self._wrap_fn(name, real)
            monkeypatch.setattr(ops, name, wrapped)
        if hasattr(ops, '_stream'):
            orig = ops._stream

            def _stream():
                if self.depth == 0:
                    self.unfaked.append(sys._getframe(1).f_code.co_name)
                return orig()
            monkeypatch.setattr(ops, '_stream', _stream)

    # ------------------------------------------------------------------ wrapping
    def _inside(self, fn, *a, **k):
        self.depth += 1
        try:
            return fn(*a, **k)
        finally:
            self.depth -= 1

    def _wrap_fn(self, name, real):
        sig = inspect.signature(real)

        def wrapped(*a, **k):
            return self._call(name, sig, real, None, a, k)
        wrapped.__name__ = name
        return wrapped

    def _wrap_class(self, name, base):
        rec = self
        if name == 'GradScale':
            class Rec(base):
                def from_amax(s, a, b=None, target=None):
                    return rec._call('GradScale', inspect.signature(base.from_amax), base.from_amax, s,
                                     (a, b, target), {})
            return Rec

        class Rec(base):
            def __init__(s, *a, **k):
                rec._inside(super().__init__, *a, **k)

            def refresh(s, weight, bias=None, force=False):
                if name == 'PackedConv':
                    rec._inside(super().refresh, weight, bias, force)
                else:
                    rec._inside(super().refresh, weight, force)
                rec.params[id(s)] = (weight.detach().float().cpu().clone(),
                                     bias.detach().float().cpu().clone() if bias is not None else None)
                rec.layers[id(s)] = s

            def __call__(s, *a, **k):
                return rec._call(name, inspect.signature(base.__call__), base.__call__, s, a, k)
        Rec.__name__ = base.__name__
        return Rec

    # ------------------------------------------------------------------ stand-ins of the layer objects
    def _fake_conv(self, pc, absolute=False, epilogue=None):
        w, b = self.params[id(pc)]
        w = w.half().to(F64)
        b = b.to(F64)
        if absolute:
            w, b = w.abs(), b.abs()
        with _Mode():
            return FK.PackedConv(w, b, pc.kind, pc.act, pc.epilogue if epilogue is None else epilogue)

    def _fake_dgrad(self, pd, absolute=False):
        w, _ = self.params[id(pd)]
        w = w.half().to(F64)
        with _Mode():
            return FK.PackedDgrad(self._fake_conv(pd.fwd, absolute), w.abs() if absolute else w)

    @staticmethod
    def _fake_scale(ws):
        s = FK.GradScale(None)
        s.ws = ws.detach().cpu().float().clone()
        return s

    # ------------------------------------------------------------------ one call
    def _call(self, name, sig, real, obj, a, k):
        self.seen.add(name)
        if self.depth:
            return real(obj, *a, **k) if obj is not None else real(*a, **k)
        ba = sig.bind(*((obj,) if obj is not None else ()), *a, **k)
        ba.apply_defaults()
        args = dict(ba.arguments)
        args.pop('self', None)
        for p in sig.parameters.values():       # a stand-in taking **kw: its keywords are arguments like the others
            if p.kind == p.VAR_KEYWORD:
                args.update(args.pop(p.name, {}))
        snap = {key: (v.detach().cpu().clone() if isinstance(v, torch.Tensor) else v) for key, v in args.items()}
        scale = args.get('scale')
        scale_ws = scale.ws.detach().cpu().clone() if scale is not None and hasattr(scale, 'ws') else None
        ins = [v for key, v in args.items() if isinstance(v, torch.Tensor) and key not in OUTPUTS[name]]
        for key in OUTPUTS[name]:
            t = args.get(key)
            accumulating = (name, key) in ACCUMULATING or (key in ('y', 'gx') and args.get('accumulate'))
            if isinstance(t, torch.Tensor) and not accumulating and not any(_overlaps(t, i) for i in ins):
                _poison(t)
        out = self._inside(real, obj, *a, **k) if obj is not None else self._inside(real, *a, **k)
        self._check(name, obj, args, snap, scale_ws, out)
        return out

    def _ref_args(self, name, obj, snap, scale_ws, absolute):
        r = {}
        for key, v in snap.items():
            if isinstance(v, torch.Tensor) and v.is_floating_point():
                v = v.to(F64)
                r[key] = v.abs() if absolute else v
            elif key == 'mul' and absolute:
                r[key] = abs(v)
            elif key in ('fwd', 'up', 'outc'):
                r[key] = self._fake_conv(v, absolute)
            elif key == 'scale' and hasattr(v, 'ws'):
                r[key] = self._fake_scale(scale_ws)
            else:
                r[key] = v
        if name == 'PackedConv':
            fake = self._fake_conv(obj, absolute, FK.EPI_OUT_NCHW_F32 if absolute and obj.epilogue == FK.EPI_FLOW_NCHW_F32
                                   else None)
            return (lambda **kw: fake(**kw)), r
        if name == 'PackedDgrad':
            fake = self._fake_dgrad(obj, absolute)
            return (lambda **kw: fake(**kw)), r
        if name == 'GradScale':
            fake = self._fake_scale(scale_ws if scale_ws is not None else obj.ws)
            return (lambda **kw: fake.from_amax(**kw)), r
        return getattr(FK, name), r

    @staticmethod
    def _collect(name, out, args):
        """{output name: tensor} of one call (return value and written arguments)"""
        res = {}
        written = [args.get(key) for key in OUTPUTS[name] if isinstance(args.get(key), torch.Tensor)]
        for key in OUTPUTS[name]:
            if isinstance(args.get(key), torch.Tensor):
                res[key] = args[key]
        if isinstance(out, tuple):
            for i, t in enumerate(out):
                if isinstance(t, torch.Tensor):
                    res[f'ret{i}'] = t
        elif isinstance(out, torch.Tensor) and not any(out is t or (out.data_ptr() == t.data_ptr() and
                                                                    out.shape == t.shape) for t in written):
            res['ret'] = out
        return res

    def _check(self, name, obj, args, snap, scale_ws, out):
        got = {key: t.detach().cpu() for key, t in self._collect(name, out, args).items()}
        fn, ra = self._ref_args(name, obj, snap, scale_ws, False)
        bounds = None
        if name == 'fused_tail':
            ref, bounds = self._tail(ra)
        else:
            with _Mode():
                rout = fn(**ra)
            ref = {key: t for key, t in self._collect(name, rout, ra).items()}
        msgs = []
        if name in ('GradScale', 'flow_head_bwd'):
            ws_got = (obj if name == 'GradScale' else args['scale']).ws.detach().cpu().float()[:2]
            ws_ref = (rout if name == 'GradScale' else ra['scale']).ws.float()[:2]
            if not torch.equal(ws_got, ws_ref):
                msgs.append(f'loss scale {ws_got.tolist()} != {ws_ref.tolist()}')
        worst = 0.0
        if name in EXACT:
            for key, g in got.items():
                r = ref[key].to(g.dtype)
                ib = {torch.float16: torch.int16, torch.uint8: torch.uint8}.get(g.dtype, torch.int32)
                if g.shape != r.shape or not torch.equal(g.contiguous().view(ib), r.contiguous().view(ib)):
                    bad = int((g.double() != r.double()).sum()) if g.shape == r.shape else -1
                    msgs.append(f'{key}: not bit-exact ({bad} elements differ)')
                    worst = float('inf')
        else:
            if bounds is None:
                bounds = self._bounds(name, obj, args, snap, scale_ws, fn, ra, ref,
                                      {key: g.dtype for key, g in got.items()})
            for key, g in got.items():
                if name == 'fused_tail' and key == 'y_u8':
                    # the uint8 frame is float32_to_uint8 of the kernel's OWN fp32 frame, bit for bit; how far that
                    # frame is from the reference is the y check's business
                    want = FK.float_to_uint8_nhwc(got['y'])
                    if not torch.equal(g, want):
                        msgs.append(f'y_u8: not float32_to_uint8(y) ({int((g != want).sum())} elements differ)')
                        worst = float('inf')
                    continue
                r = ref[key]
                gd = g.double()
                if gd.shape != r.shape:
                    msgs.append(f'{key}: shape {tuple(gd.shape)} != {tuple(r.shape)}')
                    continue
                bound = bounds[key]
                err = (gd - r).abs()
                err = torch.where(torch.isnan(gd), torch.full_like(err, float('inf')), err)
                ratio = torch.where(bound > 0, err / bound, torch.where(err > 0, float('inf'), 0.0))
                m = float(ratio.max()) if ratio.numel() else 0.0
                worst = max(worst, m)
                if m > 1.0:
                    idx = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
                    msgs.append(f'{key}: |err| {float(err[idx]):.3e} > bound {float(bound[idx]):.3e} at {idx} '
                                f'(got {float(gd[idx])!r}, ref {float(r[idx])!r})')
        self.calls[name] = self.calls.get(name, 0) + 1
        self.worst[name] = max(self.worst.get(name, 0.0), worst)
        if msgs:
            shapes = {key: tuple(v.shape) for key, v in snap.items() if isinstance(v, torch.Tensor)}
            self.failures.append(f'{name} {shapes}: ' + '; '.join(msgs))

    # ------------------------------------------------------------------ bounds
    def _bounds(self, name, obj, args, snap, scale_ws, fn, ra, ref, dtypes):
        """{output: per-element bound} of an arithmetic op: ulp_out(ref) + gamma_K * (the op on |operands|)"""
        fa, aa = self._ref_args(name, obj, snap, scale_ws, True)
        if name == 'PackedConv' and args.get('pool'):
            # pooled epilogue: the bound of the unpooled conv, max-pooled over the same 2x2 windows.  Each pooled
            # output is max_i a_i (kernel) against max_i b_i (reference) over one window, and
            # |max_i a_i - max_i b_i| <= max_i |a_i - b_i| <= max_i bound_i
            key, = ref
            ra, aa = dict(ra, pool=False, y=None), dict(aa, pool=False, y=None)
            with _Mode():
                r = fn(**ra)
            with _Mode(absolute=True):
                a = fa(**aa)
            b = self._bound(name, key, obj, args, ra, r, a, dtypes[key])
            return {key: F.max_pool2d(b.permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1)}
        if name == 'flow_head_bwd':        # |terms| of g * (24 - f^2/24): |g| * 48, times the chosen scale
            aa['flow'] = torch.zeros_like(aa['flow'])
        with _Mode(absolute=True):
            aout = fa(**aa)
        absop = self._collect(name, aout, aa)
        if name == 'flow_head_bwd':
            s = float(ra['scale'].ws[0])
            g = (ra['gflow'].abs() + (ra['gflow2'].abs() if ra['gflow2'] is not None else 0)) * 48 * s
            key, = ref
            a = torch.zeros(ref[key].shape, dtype=F64)
            a[..., :2] = g.permute(0, 2, 3, 1)
            absop = {key: a}
        return {key: self._bound(name, key, obj, args, ra, r, absop[key], dtypes[key])
                for key, r in ref.items() if key in dtypes}

    def _bound(self, name, key, obj, args, ra, r, a, dtype):
        k = gamma(self._k(name, key, obj, args))
        if name == 'PackedConv' and obj.epilogue == FK.EPI_FLOW_NCHW_F32:    # 24 * tanhf(pre-activation)
            return 4 * ulp(r, dtype) + 24 * k * a
        return ulp(r, dtype) + k * a + self._extra(name, key, ra, r, dtype)

    @staticmethod
    def _tail(ra):
        """fused_tail: the float64 reference of y and its bound, one image at a time (the 64-channel HR map of a
        bench frame is 350 MB in float64).  With t = relu(convT(x) + b_up) >= 0 and r the residual (the pre-written y when
        accumulating, else upsample_func(lr_curr)):
          * the kernel sums convT in fp32 and keeps the 64-channel HR map in fp16:
              |t_k - t| <= e_t = gamma(K1) A1 + ulp16(|t| + gamma(K1) A1),  A1 = |b_up| + convT(|x|, |w_up|),
              K1 = 9 * 64 + 2 (relu is 1-Lipschitz);
          * then conv_out(t_k) + b_out + r in fp32, rounded to the fp32 output:
              |y_k - y| <= ulp32(y) + gamma(K2) A2 + conv_out(e_t, |w_out|),
              A2 = |b_out| + conv_out(|t| + e_t, |w_out|) + |r|,  K2 = 9 * 64 + 2 + 20 (the in-kernel bicubic
              residual is a 16-tap sum);
            the last term is the fp16 rounding of the HR map pushed through |w_out|."""
        up, outc, x, lr = ra['up'], ra['outc'], ra['x'], ra['lr_curr']
        acc = ra['accumulate']
        g1, g2 = gamma(9 * up.cin_real + 2), gamma(9 * outc.cin_real + 2 + 20)
        ys, bounds = [], []
        for i in range(x.shape[0]):
            xi = x[i:i + 1]
            lri = lr[i:i + 1] if lr is not None else None
            with _Mode():
                y = FK.fused_tail(up, outc, xi, lri, ra['lr_scale'], ra['up_mode'],
                                  y=ra['y'][i:i + 1].clone() if acc else None, accumulate=acc)
                xn = FK.to_nchw(xi, up.cin_real)
                t = F.relu(F.conv_transpose2d(xn, up.w, up.b, 2, 1, output_padding=1))
                a1 = F.conv_transpose2d(xn.abs(), up.w.abs(), up.b.abs(), 2, 1, output_padding=1)
                e_t = g1 * a1 + ulp(t + g1 * a1, torch.float16)
                wo = outc.w.abs()
                a2 = F.conv2d(t + e_t, wo, outc.b.abs(), 1, 1)
                if acc:
                    a2 = a2 + ra['y'][i:i + 1].abs()
                elif lri is not None:
                    with _Mode(absolute=True):
                        a2 = a2 + FK._up(lri.abs(), ra['lr_scale'], ra['up_mode'])
                bounds.append(ulp(y, torch.float32) + g2 * a2 + F.conv2d(e_t, wo, None, 1, 1))
            ys.append(y)
        key = 'y' if ra['y'] is not None else 'ret'
        return {key: torch.cat(ys)}, {key: torch.cat(bounds)}

    @staticmethod
    def _k(name, key, obj, args):
        """number of addends per output element (an upper bound)"""
        if name == 'PackedConv':
            return 9 * obj.cin_real + 2
        if name == 'PackedDgrad':
            return 9 * obj.fwd.cout_real + 2
        if name in ('wgrad', 'bias_grad'):
            dz = args['dz']
            return dz.shape[0] * dz.shape[1] * dz.shape[2] + 1
        if name == 'upsample':
            return 20
        if name == 'upsample_bwd':
            return 32 * args['scale_factor'] + 4
        if name == 'upsample2x':
            return 6
        if name == 'upsample2x_bwd':
            return 18
        if name == 'maxpool2x2_bwd':
            return 2
        if name == 'flow_head_bwd':
            return 8
        if name in ('warp_s2d_concat_bwd', 'backward_warp_bwd'):
            return 256 if key in ('d_hr_prev', 'ret0') else 3 * _channels(name, args) + 8
        return 8                                  # bilinear samples

    @staticmethod
    def _extra(name, key, ra, ref, dtype):
        """the bilinear warps: the kernels round the sample coordinate X + flow to fp32 (the stand-in does not)"""
        if name not in WARPS:
            return 0.0
        dflow = 0.0
        if name == 'warp_s2d_concat_lrflow':
            # the HR flow is itself computed in the kernel: scale * (an fp32 sum of <= 20 products) of the
            # reflect-padded LR flow, off by at most scale * gamma(20) * upsample_func(|lr_flow|) -- one more
            # coordinate error
            s, hw = ra['scale'], tuple(ra['lr_curr'].shape[2:])
            with _Mode():
                flow = s * FK._up(FK._reflect_pad(ra['lr_flow'], hw), s, ra['up_mode'])
            with _Mode(absolute=True):
                dflow = s * gamma(20) * float(FK._up(FK._reflect_pad(ra['lr_flow'].abs(), hw), s, ra['up_mode']).max())
        else:
            flow = ra['hr_flow'] if 'hr_flow' in ra else ra['flow']
        x = ra['hr_prev'] if 'hr_prev' in ra else ra['x']
        H, W = flow.shape[2], flow.shape[3]
        dc = 8 * U * (max(H, W) + float(flow.abs().max())) + dflow
        xmax = float(x.abs().max())
        if name in ('warp_s2d_concat_hrflow', 'warp_s2d_concat_lrflow', 'backward_warp'):
            return (gamma(8) + 2 * dc) * 4 * xmax
        g = _warp_grad_in(name, ra)                   # [n,C,H,W] gradient arriving at each HR sample
        if key in ('d_hr_flow', 'ret1'):
            return (gamma(3 * x.shape[1] + 8) + 2 * dc) * 4 * xmax * g.abs().sum(1, keepdim=True).expand_as(ref)
        return 4 * dc * _corner_scatter(g.abs(), flow)


def _channels(name, args):
    return args['hr_prev'].shape[1] if name == 'warp_s2d_concat_bwd' else args['x'].shape[1]


def _warp_grad_in(name, ra):
    if name == 'backward_warp_bwd':
        return ra['gy']
    c, s = ra['hr_prev'].shape[1], ra['scale_factor']
    with _Mode():
        g = FK.to_nchw(ra['gx'], (s * s + 1) * c)[:, c:] / FK._s(ra['scale'])
        return FK.depth_to_space(g, s)


def _corner_scatter(g, flow):
    """sum of g over every sample whose 2x2 bilinear footprint touches each element (weights 1)"""
    n, c, H, W = g.shape
    X = torch.arange(W, dtype=F64).view(1, 1, W) + flow[:, 0]
    Y = torch.arange(H, dtype=F64).view(1, H, 1) + flow[:, 1]
    xa = X.clamp(0, W - 1).floor().clamp(max=W - 2).long()
    ya = Y.clamp(0, H - 1).floor().clamp(max=H - 2).long()
    out = torch.zeros(n, c, H * W, dtype=F64)
    src = g.to(F64).reshape(n, c, H * W)
    for dy in (0, 1):
        for dx in (0, 1):
            idx = ((ya + dy) * W + xa + dx).reshape(n, 1, H * W).expand(n, c, H * W)
            out.scatter_add_(2, idx, src)
    return out.view(n, c, H, W)


# ---------------------------------------------------------------------------------------------- scenarios
def _rand(seed, *shape, lo=0.0, hi=1.0, dev='cpu'):
    return torch.from_numpy(np.random.default_rng(seed).uniform(lo, hi, size=shape).astype(np.float32)).to(dev)


def run_sequence(T, dev, seed, nb, n, t, h, w, degradation='BD', scale=4, flow_losses=True, loss_mul=1.0, nc=3):
    """one training step of FRNet.forward_sequence of an nc-channel net: loss on hr_data (and hr_flow / lr_flow),
    backward"""
    from oracle import frnet_oracle as O
    net = T.FRNet(nc, nc, 64, nb, degradation, scale)
    net.load_state_dict(O.make_frnet_params(seed, in_nc=nc, out_nc=nc, nb=nb, scale=scale, degradation=degradation,
                                            gain=1.5), strict=True)
    net = net.to(dev).train()
    d = net(_rand(seed + 1, n, t, nc, h, w, dev=dev))
    keys = ('hr_data', 'hr_flow', 'lr_flow') if flow_losses else ('hr_data',)
    loss = sum((d[k] * _rand(seed + 2 + i, *d[k].shape, lo=-1, hi=1, dev=dev)).sum() for i, k in enumerate(keys))
    (loss * loss_mul).backward()
    return net


def run_module_ops(T, ops, dev, seed):
    """net.fnet, backward_warp (flows far past the borders), upsample_func and space_to_depth under autograd,
    and the ops the training step only reaches with other arguments: an accumulating upsample_bwd with a
    negative multiplier, bias_grad into a pre-filled db, maxpool2x2_bwd over windows with tied maxima"""
    from oracle import frnet_oracle as O
    net = T.FRNet(3, 3, 64, 1, 'BD', 4)
    net.load_state_dict(O.make_frnet_params(seed, nb=1, gain=1.5), strict=True)
    net = net.to(dev).train()
    x1, x2 = _rand(seed + 1, 2, 3, 16, 24, dev=dev), _rand(seed + 2, 2, 3, 16, 24, dev=dev)
    (net.fnet(x1, x2) * _rand(seed + 3, 2, 2, 16, 24, lo=-1, hi=1, dev=dev)).sum().backward()
    a = _rand(seed + 4, 2, 3, 12, 20, dev=dev).requires_grad_(True)
    f = _rand(seed + 5, 2, 2, 12, 20, lo=-30, hi=30, dev=dev).requires_grad_(True)
    (T.backward_warp(a, f) * _rand(seed + 6, 2, 3, 12, 20, lo=-1, hi=1, dev=dev)).sum().backward()
    b = _rand(seed + 7, 2, 3, 5, 9, dev=dev).requires_grad_(True)
    (net.upsample_func(b) * _rand(seed + 8, 2, 3, 20, 36, lo=-1, hi=1, dev=dev)).sum().backward()
    c = _rand(seed + 9, 1, 3, 8, 12, dev=dev).requires_grad_(True)
    (T.space_to_depth(c, 4) * _rand(seed + 10, 1, 48, 2, 3, lo=-1, hi=1, dev=dev)).sum().backward()
    gx = _rand(seed + 11, 1, 2, 5, 9, lo=-1, hi=1, dev=dev)
    ops.upsample_bwd(_rand(seed + 12, 1, 2, 20, 36, lo=-1, hi=1, dev=dev), 4, FK.UP_BICUBIC, mul=-0.5, gx=gx,
                     accumulate=True)
    dz = _rand(seed + 13, 3, 7, 5, 64, lo=-4, hi=4, dev=dev).half()
    ops.bias_grad(dz, _rand(seed + 14, 48, lo=-1, hi=1, dev=dev))
    rng = np.random.default_rng(seed + 15)
    x = torch.from_numpy(rng.choice(np.array([-1.0, -0.0, 0.0, 0.5, 2.0], np.float16), size=(2, 6, 8, 64))).to(dev)
    ops.maxpool2x2_bwd(x, _rand(seed + 16, 2, 3, 4, 64, lo=-1, hi=1, dev=dev).half(), FK.ACT_LRELU02)


def scenarios(T, ops, dev):
    """the replay of the training path: bd4 with hr_flow / lr_flow losses (gflow2, the caller's hr_flow gradient,
    n*t batched wgrad), bd4 at the product depth with a 1e-7 loss (the loss-scale regime), bi2, module ops"""
    run_sequence(T, dev, 31, nb=2, n=2, t=4, h=32, w=32)
    run_sequence(T, dev, 32, nb=10, n=1, t=3, h=32, w=32, flow_losses=False, loss_mul=1e-7)
    run_sequence(T, dev, 33, nb=1, n=1, t=3, h=16, w=24, degradation='BI', scale=2)
    run_module_ops(T, ops, dev, 34)


# ---------------------------------------------------------------------------------------------- inference scenarios
def inference_ops(tail, pool):
    """the ops FRNet.step_into launches with ops.tail_mode() == tail and ops.pool_fused() == pool"""
    names = {'pack_pair', 'PackedConv', 'upsample2x', 'warp_s2d_concat_lrflow'}
    if not pool:
        names.add('maxpool2x2')
    if tail in ('acc', 'fused'):
        names.add('fused_tail')
    if tail != 'fused':
        names |= {'upsample', 'float_to_uint8_nhwc'}
    return names


def run_frames(T, net, clips, dev):
    """the recurrent eval step over clips [n,t,c,h,w] (c = the net's in_nc) from zero state -- ClipEngine.run_frame without a CUDA graph on
    a GPU (the step bench.py times), FRNet.step_into with a uint8 output on the CPU.  Returns the last (hr, u8)."""
    n, t, c, h, w = clips.shape
    s = net.scale
    if torch.device(dev).type == 'cuda':
        eng = T.ClipEngine(net, n, c, h, w, dev, use_graph=False)
        eng.reset()
        for i in range(t):
            eng.lr[i & 1].copy_(clips[:, i].to(dev))
            eng.run_frame(i & 1)
        torch.cuda.synchronize()
        return eng.hr[(t - 1) & 1], eng.u8[(t - 1) & 1]
    lr_prev, hr_prev = torch.zeros(n, c, h, w), torch.zeros(n, c, s * h, s * w)
    for i in range(t):
        lr = clips[:, i].contiguous()
        hr, u8 = torch.empty(n, c, s * h, s * w), torch.empty(n, s * h, s * w, c, dtype=torch.uint8)
        net.step_into(lr, lr_prev, hr_prev, hr, out_u8=u8)
        lr_prev, hr_prev = lr, hr
    return hr, u8


def run_inference(T, ops, dev, seed, nb, n, t, h, w, degradation='BD', scale=4, params=None, clips=None, nc=3):
    """t recurrent eval steps of n lock-stepped clips of nc x h x w (O.make_clip, or `clips` [n,t,nc,h,w]) through an
    nc-channel net with O.make_frnet_params(gain=1.5) (or `params`).  The net is built here, after the Recorder is
    installed: layer objects made earlier would bypass its wrapped classes."""
    from oracle import frnet_oracle as O
    net = T.FRNet(nc, nc, 64, nb, degradation, scale)
    if params is None:
        params = O.make_frnet_params(seed, in_nc=nc, out_nc=nc, nb=nb, scale=scale, degradation=degradation, gain=1.5)
    net.load_state_dict(params, strict=True)
    net = net.to(dev).eval()
    if clips is None:
        clips = torch.stack([O.make_clip(seed + 1 + k, t, nc, h, w) for k in range(n)])
    return run_frames(T, net, clips, dev)


def run_inference_module_ops(T, ops, dev, seed):
    """the inference ops at edges the product step rarely reaches: warp_s2d_concat_lrflow on uniform-noise hr_prev
    with LR flows of +-30 px (far past the borders) at sizes that are not multiples of 8 (reflect pad), bicubic x4
    and bilinear x2; float_to_uint8_nhwc on values out of range and on exact rounding ties"""
    for i, (scale, mode, h, w) in enumerate(((4, FK.UP_BICUBIC, 13, 22), (2, FK.UP_BILINEAR, 11, 19))):
        s = seed + 10 * i
        ops.warp_s2d_concat_lrflow(_rand(s, 2, 3, scale * h, scale * w, dev=dev),
                                   _rand(s + 1, 2, 2, h // 8 * 8, w // 8 * 8, lo=-30, hi=30, dev=dev),
                                   _rand(s + 2, 2, 3, h, w, dev=dev), scale, mode)
    rng = np.random.default_rng(seed + 30)
    ties = (rng.integers(-3, 259, size=(2, 3, 7, 11)) + 0.5) / 255.0
    x = np.where(rng.random(ties.shape) < 0.5, ties, rng.uniform(-0.2, 1.2, size=ties.shape)).astype(np.float32)
    ops.float_to_uint8_nhwc(torch.from_numpy(x).to(dev))


def report(rec):
    return {name: (rec.calls.get(name, 0), round(rec.worst.get(name, 0.0), 4)) for name in sorted(rec.calls)}
