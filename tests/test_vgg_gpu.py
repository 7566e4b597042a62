"""GPU tests of the VGG19 perceptual-loss path: the 512-channel conv and dgrad (wgmma against the CUDA-core kernel per
element, and that against float64), each feature and the input gradient of the cosine feature loss against float64
autograd, the gt pass without a tape, determinism, guard bands around the new kernels' outputs, the new packing calls
replayed against their contracts, and the reference's VSRGANModel.train() with this extractor as net_F."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

import tecogan_b200 as T                            # noqa: E402
import refimport                                    # noqa: E402

ops = T.ops
L = sys.modules['tecogan-pytorch_b200.lib']
pytestmark = pytest.mark.gpu
DEV = torch.device('cuda', 0)
F64 = torch.float64
# Bounds against float64 (DESIGN.md section 10), from the errors measured on an H100 with a margin:
#   features: rel-L2 FEAT_REL[index], SURVEY 8(d)'s 1e-3 for relu2_2 and relu3_4; relu4_4 and relu5_4 measured
#     1.04e-3 and 1.16e-3: the fp16 rounding of the weights and of every layer's stored output compounds over 12 and
#     16 convs, so they get 2e-3;
#   input gradient of the cosine feature loss: GRAD_REL against float64 autograd whose ReLUs and max-pools take the
#     decisions the kernels' forward took (which elements pass, which element of each window); against plain float64,
#     GRAD_REL where no max-pool lies on the backward path (relu1_2 alone, measured 6.7e-3) and GRAD_REL_POOLED through
#     the pools (measured 7.6e-2): an element whose pre-activation lies within the fp16 path's error of 0, or a window
#     whose two largest inputs lie within fp16's spacing, passes or routes its gradient differently than float64 does,
#     and that moves a whole element of the gradient (4.8e-2 with the pool routes alone made equal).
FEAT_REL = {1: 1e-3, 3: 1e-3, 8: 1e-3, 17: 1e-3, 26: 2e-3, 35: 2e-3}
GRAD_REL, GRAD_REL_POOLED = 1e-2, 1.2e-1


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


@pytest.fixture(scope='module', autouse=True)
def seeded_vgg19():
    refimport.stub_pretrained_vgg19()


@pytest.fixture(scope='module')
def vgg():
    return T.VGGFeatureExtractor().to(DEV)


# ------------------------------------------------------------------ the 512-channel conv and dgrad
CONV_CASES = [(512, 512), (256, 512), (512, 256), (3, 512), (500, 512)]
SIZES = [(1, 16, 8), (1, 17, 9), (2, 31, 77), (1, 5, 3)]


def _layer(cin_real, cout, seed):
    g = torch.Generator().manual_seed(seed)
    wt = torch.randn(cout, cin_real, 3, 3, generator=g) / (3 * cin_real ** 0.5)
    b = torch.randn(cout, generator=g) * 0.1
    return wt, b, g


@pytest.mark.parametrize('cin_real,cout', CONV_CASES)
@pytest.mark.parametrize('n,h,w', SIZES)
def test_512_channel_conv_matches_simt_and_float64(cin_real, cout, n, h, w):
    wt, b, g = _layer(cin_real, cout, cin_real * 1000 + cout + h)
    cin = ops.pad64(cin_real)
    x = torch.randn(n, h, w, cin, generator=g).half()
    x[..., cin_real:] = 0
    conv = ops.PackedConv(wt.to(DEV), b.to(DEV), L.CONV_3X3, L.ACT_RELU, L.EPI_NHWC_F16)
    xd = x.to(DEV)
    y_tc, y_simt = conv(xd, impl='tcgen05'), conv(xd, impl='simt')
    torch.cuda.synchronize()
    xs = x[..., :cin_real].to(DEV, F64).permute(0, 3, 1, 2)
    ref = F.relu(F.conv2d(xs, wt.half().to(DEV, F64), b.to(DEV, F64), padding=1)).permute(0, 2, 3, 1)
    d = (y_tc.float() - y_simt.float()).abs()
    assert bool((d <= 2e-3 * (1 + y_simt.float().abs())).all()), float(d.max())
    assert _rel(y_simt, ref) <= 1e-3


@pytest.mark.parametrize('cin_real,cout', CONV_CASES)
@pytest.mark.parametrize('n,h,w', SIZES)
def test_512_channel_dgrad_with_mask_and_residual_matches_simt_and_float64(cin_real, cout, n, h, w):
    wt, b, g = _layer(cin_real, cout, cin_real * 1000 + cout + h + 7)
    cin = ops.pad64(cin_real)
    fwd = ops.PackedConv(wt.to(DEV), b.to(DEV), L.CONV_3X3, L.ACT_RELU, L.EPI_NHWC_F16)
    dg = ops.PackedDgrad(fwd, wt.to(DEV))
    dz = torch.randn(n, h, w, cout, generator=g).half()
    res = torch.randn(n, h, w, cin, generator=g).half()
    res[..., cin_real:] = 0
    mask = torch.randn(n, h, w, cin, generator=g).half()
    args = [t.to(DEV) for t in (dz, res, mask)]
    y_tc = dg(args[0], residual=args[1], mask=args[2], mask_act=L.ACT_RELU, impl='tcgen05')
    y_simt = dg(args[0], residual=args[1], mask=args[2], mask_act=L.ACT_RELU, impl='simt')
    torch.cuda.synchronize()
    gx = F.conv_transpose2d(dz.to(DEV, F64).permute(0, 3, 1, 2), wt.half().to(DEV, F64), padding=1).permute(0, 2, 3, 1)
    gx = F.pad(gx, (0, cin - cin_real))
    ref = (gx + res.to(DEV, F64)) * (mask.to(DEV, F64) > 0)
    d = (y_tc.float() - y_simt.float()).abs()
    assert bool((d <= 2e-3 * (1 + y_simt.float().abs())).all()), float(d.max())
    assert _rel(y_simt, ref) <= 1e-3
    assert bool((y_tc[..., cin_real:] == 0).all())


# ------------------------------------------------------------------ features and input gradient against float64
def _ref_features(vgg, x, routes=None):
    """the reference's forward in float64 on the device, up to the deepest requested index.  routes (_routes): the
    discontinuities as the kernels' forward took them: each ReLU keeps the elements the kernels' stored output has
    positive, each max-pool takes the element of each window the kernels' pool took (the gradient then follows the
    same masks and routes)"""
    out, feats = (x.to(F64) - vgg.mean.to(F64)) / vgg.std.to(F64), []
    for i in range(max(vgg.feature_indexs) + 1):
        m = vgg.features[i]
        if isinstance(m, torch.nn.Conv2d):
            out = F.conv2d(out, m.weight.to(F64), m.bias.to(F64), padding=1)
        elif isinstance(m, torch.nn.ReLU):
            out = F.relu(out) if routes is None else out * routes[i]
        elif routes is not None:
            out = torch.gather(_windows(out), -1, routes[i].unsqueeze(-1)).squeeze(-1)
        else:
            out = F.max_pool2d(out, 2, 2)
        if i in vgg.feature_indexs:
            feats.append(out)
    return feats


def _windows(t):
    """NCHW [N,C,H,W] -> [N,C,H/2,W/2,4], the 2x2 windows of the floor pool in row-major order"""
    n, c, h, w = t.shape
    t = t[:, :, :h // 2 * 2, :w // 2 * 2].reshape(n, c, h // 2, 2, w // 2, 2)
    return t.permute(0, 1, 2, 4, 3, 5).reshape(n, c, h // 2, w // 2, 4)


def _routes(vgg, x):
    """the kernels' forward decisions: {ReLU index: stored output > 0, max-pool index: the first maximum of each
    window of the stored fp16 ReLU output}"""
    A = sys.modules['tecogan-pytorch_b200.autograd']
    with torch.no_grad():
        _, outs = A.vgg_forward(vgg, x.contiguous(), keep=True)
    r = {}
    for (ci, ri, pool), a in zip(vgg._units, outs):
        a = a.permute(0, 3, 1, 2)[:, :vgg.features[ci].out_channels].float()
        r[ri] = (a > 0).to(F64)
        if pool:
            r[ci + 2] = torch.argmax(_windows(a), dim=-1)
    return r


def _cos_loss(hr_feats, gt_feats):
    return sum(1.0 - F.cosine_similarity(a, b.detach(), dim=1, eps=1e-8).mean() for a, b in zip(hr_feats, gt_feats))


def _pair(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    gt = torch.rand(n, 3, h, w, generator=g)
    hr = (gt + 0.1 * torch.randn(n, 3, h, w, generator=g)).clamp(0, 1)
    return hr.to(DEV), gt.to(DEV)


@pytest.mark.parametrize('n,h,w', [(4, 64, 64), (1, 256, 256), (2, 70, 90)])
def test_features_against_float64(vgg, n, h, w):
    _, x = _pair(n, h, w, h + w)
    with torch.no_grad():
        got = vgg(x)
        want = _ref_features(vgg, x)
    assert len(got) == 4
    for k, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == torch.float32 and tuple(a.shape) == tuple(b.shape), k
        e = _rel(a, b)
        print(f'feature {vgg.feature_indexs[k]} {n}x{h}x{w}: rel-L2 {e:.2e}')
        assert e <= FEAT_REL[vgg.feature_indexs[k]], (k, e)


@pytest.mark.parametrize('idx', [(8, 17, 26, 35), (3,)])
@pytest.mark.parametrize('n,h,w,loss_mul', [(4, 64, 64, 1.0), (2, 70, 90, 1.0), (4, 64, 64, 1e-6)])
def test_input_gradient_against_float64(n, h, w, loss_mul, idx):
    """loss_mul = 1e-6 puts the relu2_2 gradient at ~1e-9 per element, below the training shape's ~1e-7: the loss
    scale has to bring it into fp16's range"""
    vgg = T.VGGFeatureExtractor(idx).to(DEV)
    hr, gt = _pair(n, h, w, 3 * h + w)
    x = hr.clone().requires_grad_(True)
    with torch.no_grad():
        gt_feats = vgg(gt)
    loss = _cos_loss(vgg(x), gt_feats) * loss_mul
    g_ours, = torch.autograd.grad(loss, [x])
    errs = []
    for routes in (_routes(vgg, hr), None):
        x64 = hr.to(F64).requires_grad_(True)
        with torch.no_grad():
            gt64 = _ref_features(vgg, gt)
        g_ref, = torch.autograd.grad(_cos_loss(_ref_features(vgg, x64, routes), gt64) * loss_mul, [x64])
        errs.append(_rel(g_ours, g_ref))
    print(f'input gradient {idx} {n}x{h}x{w} loss x {loss_mul}: rel-L2 {errs[0]:.2e} (float64, the kernels\' ReLU '
          f'masks and pool routes), {errs[1]:.2e} (float64)')
    assert errs[0] <= GRAD_REL, errs
    assert errs[1] <= (GRAD_REL if idx == (3,) else GRAD_REL_POOLED), errs


def test_gt_pass_saves_nothing(vgg):
    hr, gt = _pair(2, 64, 64, 5)
    vgg(gt)                                          # warm: packed weights exist
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    torch.cuda.reset_peak_memory_stats(DEV)
    feats = vgg(gt)                                  # requires_grad=False, grad mode on: the gt pass of the loss
    torch.cuda.synchronize()
    assert all(f.grad_fn is None and not f.requires_grad for f in feats)
    held = torch.cuda.memory_allocated(DEV) - base
    assert held == sum(f.numel() * 4 for f in feats), held
    peak_nograd = torch.cuda.max_memory_allocated(DEV) - base
    del feats
    torch.cuda.reset_peak_memory_stats(DEV)
    x = hr.clone().requires_grad_(True)
    feats = vgg(x)
    torch.cuda.synchronize()
    held_grad = torch.cuda.memory_allocated(DEV) - base - x.numel() * 4
    # the hr pass keeps every conv's fp16 output as its tape; the gt pass kept none, and at no time held one
    tape, (h, w) = 0, (64, 64)
    for ci, _, pool in vgg._units:
        tape += 2 * h * w * vgg.features[ci].out_channels * 2
        if pool:
            h, w = h // 2, w // 2
    assert held_grad >= held + tape, (held_grad, held, tape)
    assert peak_nograd < held + tape
    del feats


def test_two_runs_give_the_same_bits(vgg):
    hr, gt = _pair(2, 70, 90, 11)
    res = []
    for _ in range(2):
        x = hr.clone().requires_grad_(True)
        with torch.no_grad():
            gf = vgg(gt)
        feats = vgg(x)
        g, = torch.autograd.grad(_cos_loss(feats, gf), [x])
        res.append([f.detach().clone() for f in feats] + [g])
    for a, b in zip(*res):
        assert torch.equal(a, b)


# ------------------------------------------------------------------ guard bands
def _guarded(shape, dtype):
    """a tensor of `shape` inside a 0xAB-filled buffer with 4 KB of guard on each side"""
    item = torch.empty((), dtype=dtype).element_size()
    n, g = int(np.prod(shape)), 4096 // item
    buf = torch.full(((n + 2 * g) * item,), 0xAB, dtype=torch.uint8, device=DEV)
    return buf, buf[g * item:(g + n) * item].view(dtype).view(shape), g * item, (g + n) * item


def _intact(buf, lo, hi):
    return bool((buf[:lo] == 0xAB).all()) and bool((buf[hi:] == 0xAB).all())


def test_guard_bands_of_the_new_kernels():
    n, h, w = 1, 17, 9
    wt, b, g = _layer(512, 512, 3)
    fwd = ops.PackedConv(wt.to(DEV), b.to(DEV), L.CONV_3X3, L.ACT_RELU, L.EPI_NHWC_F16)
    x = torch.randn(n, h, w, 512, generator=g).half().to(DEV)
    buf, y, lo, hi = _guarded((n, h, w, 512), torch.float16)
    fwd(x, y=y)
    bufd, yd, lod, hid = _guarded((n, h, w, 512), torch.float16)
    ops.PackedDgrad(fwd, wt.to(DEV))(x, y=yd, residual=x, mask=x, mask_act=L.ACT_RELU)
    a = torch.rand(n, 3, h, w).to(DEV)
    mean, std = torch.tensor([0.485, 0.456, 0.406], device=DEV), torch.tensor([0.229, 0.224, 0.225], device=DEV)
    bufp, yp, lop, hip = _guarded((n, h, w, 64), torch.float16)
    ops.grad_pack_ex(a, sub=mean, div=std, y=yp)
    t = torch.randn(n, 64, h, w).to(DEV)
    sc = ops.GradScale(DEV).from_amax_of([t, a])
    add, mask = torch.randn(n, h, w, 64).half().to(DEV), torch.randn(n, h, w, 64).half().to(DEV)
    bufm, ym, lom, him = _guarded((n, h, w, 64), torch.float16)
    ops.grad_pack_ex(t, scale=sc, add=add, mask=mask, mask_act=L.ACT_RELU, y=ym)
    bufu, yu, lou, hiu = _guarded((n, 3, h, w), torch.float32)
    ops.grad_unpack_ex(add, 3, std, scale=sc, y=yu)
    torch.cuda.synchronize()
    for bb, l0, h0 in ((buf, lo, hi), (bufd, lod, hid), (bufp, lop, hip), (bufm, lom, him), (bufu, lou, hiu)):
        assert _intact(bb, l0, h0)


# ------------------------------------------------------------------ the new calls against their contracts
def _ulp16(ref):
    a = ref.abs()
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -14)))
    return torch.exp2(e - 10)


def test_new_calls_of_one_forward_and_backward_against_their_contracts(vgg, monkeypatch):
    """every grad_pack_ex / grad_unpack_ex / GradScale.from_amax_of call of one hr + gt pass and the backward,
    replayed in float64 on the call's own inputs"""
    calls = []

    def rec(name, real):
        def wrapped(*a, **k):
            snap = ([t.detach().cpu().clone() if isinstance(t, torch.Tensor) else t for t in a],
                    {key: (v.detach().cpu().clone() if isinstance(v, torch.Tensor) else v) for key, v in k.items()})
            scale = k.get('scale')
            ws = scale.ws.detach().cpu().clone() if scale is not None else None
            out = real(*a, **k)
            if name == 'from_amax_of':
                ws = out.ws.detach().cpu().clone()
            calls.append((name, snap, ws, out.detach().cpu().clone() if isinstance(out, torch.Tensor) else None))
            return out
        return wrapped

    monkeypatch.setattr(ops, 'grad_pack_ex', rec('grad_pack_ex', ops.grad_pack_ex))
    monkeypatch.setattr(ops, 'grad_unpack_ex', rec('grad_unpack_ex', ops.grad_unpack_ex))
    real_amax = ops.GradScale.from_amax_of
    monkeypatch.setattr(ops.GradScale, 'from_amax_of',
                        lambda s, ts, target=None: rec('from_amax_of', lambda *a: real_amax(s, *a))(ts))
    hr, gt = _pair(2, 40, 48, 21)
    x = hr.clone().requires_grad_(True)
    with torch.no_grad():
        gf = vgg(gt)
    torch.autograd.grad(_cos_loss(vgg(x), gf), [x])
    torch.cuda.synchronize()
    names = [c[0] for c in calls]
    # two input normalisations, one scale, the deepest tap, three pooled taps, the input gradient
    assert names.count('grad_pack_ex') == 6 and names.count('from_amax_of') == 1 and names.count('grad_unpack_ex') == 1
    for name, (a, k), ws, out in calls:
        if name == 'from_amax_of':
            amax = max(float(t.abs().max()) for t in a[0])
            s = float(ws[0])
            assert s == 2.0 ** np.floor(np.log2(ops.GradScale.TARGET / amax)) and float(ws[1]) == 1.0 / s
            continue
        s = float(ws[0]) if ws is not None else 1.0
        if name == 'grad_pack_ex':
            v = a[0].to(F64)
            if k.get('sub') is not None:
                v = (v - k['sub'].to(F64).view(1, -1, 1, 1)) / k['div'].to(F64).view(1, -1, 1, 1)
            v = v * s
            v = F.pad(v.permute(0, 2, 3, 1), (0, out.shape[-1] - v.shape[1]))
            if k.get('add') is not None:
                v = v + k['add'].to(F64)
            if k.get('mask') is not None:
                v = v * (k['mask'] > 0)
            err = (out.to(F64) - v).abs()
            assert bool((err <= _ulp16(v) + 1e-6 * v.abs()).all()), float(err.max())
        else:
            x16, c, div = a[0], a[1], a[2]
            v = x16[..., :c].to(F64).permute(0, 3, 1, 2) / s / div.to(F64).view(1, -1, 1, 1)
            err = (out.to(F64) - v).abs()
            assert bool((err <= 4 * 2.0 ** -24 * v.abs()).all()), float(err.max())


# ------------------------------------------------------------------ the reference's training step
def test_reference_gan_training_with_this_net_F():
    """VSRGANModel.train() from oracle/_ref with tecogan_b200's generator and VGGFeatureExtractor on the GPU, against
    the same step with the reference generator and the reference VGG on the CPU (same weights, the shape of
    gpu_checks.check_reference_gan_training_integration)"""
    if not refimport.available():
        pytest.skip('reference not installed (oracle/_ref)')
    from oracle import frnet_oracle as O
    p = O.make_frnet_params(43, nb=2, gain=1.0)
    gt = torch.from_numpy(np.random.default_rng(80).uniform(0, 1, (1, 10, 3, 72, 72)).astype(np.float32))

    def run(device, define_generator, donor=None):
        opt = refimport.training_opt('tecogan', device=device, nb=2)
        opt['dataset']['train']['crop_size'] = 64
        m = refimport.build_training_model(opt, define_generator)
        m.net_G.load_state_dict(p, strict=True)
        if donor is not None:
            m.net_F = T.VGGFeatureExtractor(opt['train']['feature_crit']['feature_layers']).to(device)
            m.net_D.load_state_dict(donor.net_D_init)
            m.net_F.load_state_dict(donor.net_F.state_dict())
        m.net_D_init = {k: v.detach().cpu().clone() for k, v in m.net_D.state_dict().items()}
        m.prepare_training_data({'gt': gt.clone()})
        m.train()
        return m

    ref = run('cpu', None)
    got = run(DEV, T.define_generator, donor=ref)
    assert isinstance(got.net_F, T.VGGFeatureExtractor)
    losses = [k for k in ref.log_dict if k.startswith('l_')]
    assert 'l_feat_G' in losses
    for k, v in ref.log_dict.items():
        e = abs(got.log_dict[k] - v) / max(abs(v), 1e-6)
        print(f'{k}: ours {got.log_dict[k]:.6g} reference {v:.6g} rel {e:.2e}')
        # the discriminator's statistics (p_real_D, p_fake_D, distance) are not losses: they carry the generator's
        # fp16 path through the discriminator and are only printed
        assert k not in losses or e <= 3e-3, (k, got.log_dict[k], v)
    gg, rg = dict(got.net_G.named_parameters()), dict(ref.net_G.named_parameters())
    worst = max(abs(float(gg[k].grad.norm()) - float(rg[k].grad.norm())) / max(float(rg[k].grad.norm()), 1e-20)
                for k in rg)
    print(f'worst generator gradient-norm deviation {worst:.2e}')
    assert worst <= 1e-2, worst
