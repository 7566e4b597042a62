"""TEST INFRASTRUCTURE ONLY -- replays every op call of a training step against its contract in
tests/fake_ops.py, on the arguments the step actually passes.

A Recorder wraps, on the package's op layer, exactly the names fake_ops.install replaces (the PackedConv /
PackedDgrad / GradScale classes through subclasses that also note each layer's fp32 weight and bias).  For
every top-level call it

  * copies every tensor argument to the CPU before the call (in-place outputs too: dw, db, d_hr_prev, y of an
    accumulating upsample), and poisons write-only outputs with NaN;
  * runs the stand-in on those copies in float64 (weights rounded to fp16 as the kernels store them), so each
    call is judged on its own inputs and errors do not compound;
  * compares every output per element: data movement and the loss scale bit for bit; arithmetic against
    |got - ref| <= ulp_out(ref) + gamma_K * (the same op on |operands|), gamma_K = K u / (1 - K u), u = 2^-24,
    K the number of addends (plus a coordinate-rounding term for the bilinear warps).  ulp_out(0) = 0: pad
    channels and poisoned buffers must come back exactly written.

Launches through the op layer from outside a wrapped call are collected as `unfaked`, so a kernel that enters
the training path without a stand-in is reported.
"""
import inspect
import os
import sys

import numpy as np
import torch

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
}
ACCUMULATING = {('wgrad', 'dw'), ('wgrad', 'db'), ('bias_grad', 'db'), ('warp_s2d_concat_bwd', 'd_hr_prev')}
EXACT = {'pack_pair', 'nchw_to_nhwc', 'space_to_depth', 'depth_to_space', 'grad_pack', 'maxpool2x2', 'GradScale'}
WARPS = {'warp_s2d_concat_hrflow', 'warp_s2d_concat_bwd', 'backward_warp', 'backward_warp_bwd'}


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
    t.fill_(float('nan'))


class Recorder:
    def __init__(self, ops, monkeypatch):
        self.ops = ops
        self.depth = 0
        self.params = {}            # id(layer object) -> (fp32 weight, fp32 bias or None) on the CPU
        self.layers = {}            # id(layer object) -> the object (kept alive)
        self.seen = set()
        self.calls = {}             # op -> number of checked calls
        self.worst = {}             # op -> worst |err| / bound
        self.failures = []
        self.unfaked = []
        for name in FK.FAKED:
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
            elif key == 'fwd':
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
        with _Mode():
            rout = fn(**ra)
        ref = {key: t for key, t in self._collect(name, rout, ra).items()}
        msgs = []
        if name in ('GradScale', 'flow_head_bwd'):
            ws_got = (obj if name == 'GradScale' else args['scale']).ws.detach().cpu().float()[:2]
            ws_ref = (rout if name == 'GradScale' else ra['scale']).ws.float()[:2]
            if not torch.equal(ws_got, ws_ref):
                msgs.append(f'loss scale {ws_got.tolist()} != {ws_ref.tolist()}')
        if name in EXACT:
            worst = 0.0
            for key, g in got.items():
                r = ref[key].to(g.dtype)
                ib = torch.int16 if g.dtype == torch.float16 else torch.int32
                if g.shape != r.shape or not torch.equal(g.contiguous().view(ib), r.contiguous().view(ib)):
                    bad = int((g.double() != r.double()).sum()) if g.shape == r.shape else -1
                    msgs.append(f'{key}: not bit-exact ({bad} elements differ)')
                    worst = float('inf')
        else:
            fa, aa = self._ref_args(name, obj, snap, scale_ws, True)
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
            worst = 0.0
            for key, g in got.items():
                r = ref[key]
                gd = g.double()
                if gd.shape != r.shape:
                    msgs.append(f'{key}: shape {tuple(gd.shape)} != {tuple(r.shape)}')
                    continue
                bound = ulp(r, g.dtype) + gamma(self._k(name, key, obj, args)) * absop[key]
                if name == 'PackedConv' and obj.epilogue == FK.EPI_FLOW_NCHW_F32:    # 24 * tanhf(pre-activation)
                    bound = 4 * ulp(r, g.dtype) + 24 * gamma(self._k(name, key, obj, args)) * absop[key]
                bound = bound + self._extra(name, key, ra, r, g.dtype)
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
        flow = ra['hr_flow'] if 'hr_flow' in ra else ra['flow']
        x = ra['hr_prev'] if 'hr_prev' in ra else ra['x']
        H, W = flow.shape[2], flow.shape[3]
        dc = 8 * U * (max(H, W) + float(flow.abs().max()))
        xmax = float(x.abs().max())
        if name in ('warp_s2d_concat_hrflow', 'backward_warp'):
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


def run_sequence(T, dev, seed, nb, n, t, h, w, degradation='BD', scale=4, flow_losses=True, loss_mul=1.0):
    """one training step of FRNet.forward_sequence: loss on hr_data (and hr_flow / lr_flow), backward"""
    from oracle import frnet_oracle as O
    net = T.FRNet(3, 3, 64, nb, degradation, scale)
    net.load_state_dict(O.make_frnet_params(seed, nb=nb, scale=scale, degradation=degradation, gain=1.5), strict=True)
    net = net.to(dev).train()
    d = net(_rand(seed + 1, n, t, 3, h, w, dev=dev))
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


def report(rec):
    return {name: (rec.calls.get(name, 0), round(rec.worst.get(name, 0.0), 4)) for name in sorted(rec.calls)}
