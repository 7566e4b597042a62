"""pytest -m gpu: edge sweeps of the non-conv backward kernels against numpy (float64 references, or float32
emulations where the contract is bit-exact), with NaN-poisoned outputs and guard bands."""
import ctypes
import math
import os
import sys
from fractions import Fraction

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24


@pytest.fixture(scope='module')
def ops():
    import torch
    assert torch.cuda.is_available(), 'pytest -m gpu needs a GPU'
    import tecogan_b200  # noqa: F401
    return sys.modules['tecogan-pytorch_b200.ops']


def _t(a, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).to(DEV)


def _gamma(k):
    return k * U / (1 - k * U)


# ------------------------------------------------------------------------------------------ loss scale
def scale_ref(amax, target):
    """2^floor(log2(target / amax)) from exact rationals, clamped to 2^+-24; 1 for 0 / inf / NaN"""
    amax, target = float(np.float32(amax)), float(np.float32(target))
    if not (amax > 0 and math.isfinite(amax)):
        return 1.0
    q = Fraction(target) / Fraction(amax)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    return 2.0 ** max(-24, min(24, e))


def _around_powers(ks):
    out = []
    for k in ks:
        p = np.float32(2.0 ** k)
        out += [np.nextafter(p, np.float32(0)), p, np.nextafter(p, np.float32(np.inf))]
    return np.array(out, np.float32)


AMAX = _around_powers(range(-40, 41))


def _ws(sc):
    return sc.ws[:2].cpu().tolist()


@pytest.mark.parametrize('target', [256.0, 1.0, 3.0, 1000.0])
def test_loss_scale_exponent_is_exact_around_powers_of_two(ops, target):
    import torch
    sc = ops.GradScale(DEV)
    base = np.random.default_rng(1).uniform(-0.5, 0.5, 4099).astype(np.float32)
    bad = []
    for i, amax in enumerate(AMAX):
        a = base * amax                                   # every |a[j]| < amax
        a[(7 * i) % a.size] = -amax if i % 2 else amax
        got = _ws(sc.from_amax(_t(a), target=target))
        want = scale_ref(amax, target)
        if got != [want, 1.0 / want]:
            bad.append((float(amax), got[0], want))
    torch.cuda.synchronize()
    assert not bad, f'{len(bad)} wrong scales, e.g. (amax, got, want) {bad[:6]}'


@pytest.mark.parametrize('where', ['a0', 'a_last', 'b0', 'b_last', 'past_grid_cap'])
def test_loss_scale_finds_the_maximum_anywhere(ops, where):
    na = ops.sm_count() * 32 * 256 + 1000 if where == 'past_grid_cap' else 3001
    rng = np.random.default_rng(2)
    for amax in (np.float32(2.0 ** -12 * (1 + 2.0 ** -23)), np.nextafter(np.float32(2.0 ** -12), np.float32(0)),
                 np.float32(3.0), np.float32(1e-30)):
        a = (rng.uniform(-0.5, 0.5, na) * amax).astype(np.float32)
        b = (rng.uniform(-0.5, 0.5, 777) * amax).astype(np.float32)
        tgt = {'a0': (a, 0), 'a_last': (a, na - 1), 'b0': (b, 0), 'b_last': (b, b.size - 1),
               'past_grid_cap': (a, na - 1)}[where]
        tgt[0][tgt[1]] = -amax
        sc = ops.GradScale(DEV).from_amax(_t(a), _t(b))
        want = scale_ref(amax, 256.0)
        assert _ws(sc) == [want, 1.0 / want], (where, float(amax), _ws(sc), want)


@pytest.mark.parametrize('vals,want', [
    ([-0.0, -0.0, -0.0], 1.0),
    ([0.0, 0.0, 0.0], 1.0),
    ([1e-45, 0.0, -1e-45], 2.0 ** 24),
    ([1e38, -3.0, 0.0], 2.0 ** -24),
    ([float('inf'), 1.0, 0.5], 1.0),
    ([float('nan'), 1.0, 0.5], 1.0),
    ([-float('inf'), 1.0, 0.5], 1.0),
])
def test_loss_scale_special_values(ops, vals, want):
    sc = ops.GradScale(DEV).from_amax(_t(np.array(vals, np.float32)))
    assert _ws(sc) == [want, 1.0 / want]


def test_loss_scale_workspace_is_reset_between_calls(ops):
    sc = ops.GradScale(DEV)
    for amax in (1.0, 1e-3, 2.0 ** -20, 5.0):
        sc.from_amax(_t(np.array([amax, -amax / 2], np.float32)))
        want = scale_ref(amax, 256.0)
        assert _ws(sc) == [want, 1.0 / want], amax


def test_flow_head_loss_scale_and_dz_around_powers_of_two(ops):
    """flow = 0: dz = fl16(fl32(g * 24) * scale), amax = max |fl32(g * 24)|"""
    import torch
    n, h, w = 1, 4, 8
    bad = []
    for k in range(-35, 36, 1):
        c = np.float32(2.0 ** k / 24)
        for d in range(-3, 4):
            g0 = np.float32(c)
            for _ in range(abs(d)):
                g0 = np.nextafter(g0, np.float32(np.inf if d > 0 else 0))
            g = (np.random.default_rng(k + 100).uniform(-0.5, 0.5, (n, 2, h, w)) * g0).astype(np.float32)
            g[0, (k + d) % 2, d % h, 3] = -g0
            g2 = np.zeros_like(g)
            sc = ops.GradScale(DEV)
            dz = ops.flow_head_bwd(_t(g), _t(np.zeros_like(g)), sc, gflow2=_t(g2), cpad=8)
            amax = float(np.abs(g * np.float32(24)).max())
            want = scale_ref(amax, sc.TARGET)
            got = _ws(sc)
            if got != [want, 1.0 / want]:
                bad.append((amax, got[0], want))
            ref = np.zeros((n, h, w, 8), np.float16)
            ref[..., :2] = ((g * np.float32(24)) * np.float32(want)).astype(np.float16).transpose(0, 2, 3, 1)
            assert np.array_equal(dz.cpu().numpy().view(np.uint16), ref.view(np.uint16)), (k, d)
    torch.cuda.synchronize()
    assert not bad, f'{len(bad)} wrong scales, e.g. (amax, got, want) {bad[:6]}'


# ------------------------------------------------------------------------------------------ grad_pack / unpack
def _scale_obj(ops, k):
    import torch
    if k is None:
        return None, np.float32(1), np.float32(1)
    sc = ops.GradScale(DEV)
    sc.ws.copy_(torch.tensor([2.0 ** k, 2.0 ** -k, 0.0, 0.0]))
    return sc, np.float32(2.0 ** k), np.float32(2.0 ** -k)


@pytest.mark.parametrize('c,cpad', [(c, p) for c in (1, 2, 3, 51, 64, 130) for p in (8, 64, 256) if c <= p])
def test_grad_pack_and_unpack_bit_exact(ops, c, cpad):
    import torch
    rng = np.random.default_rng(c * 1000 + cpad)
    n, h, w = 2, 3, 5
    a = rng.standard_normal((n, c, h, w)).astype(np.float32) * 50
    b = rng.standard_normal((n, c, h, w)).astype(np.float32) * 50
    for use_b in (False, True):
        for k in (None, 3, -5):
            sc, s, inv = _scale_obj(ops, k)
            y = torch.full((n, h, w, cpad), float('nan'), dtype=torch.float16, device=DEV)
            ops.grad_pack(_t(a), _t(b) if use_b else None, sc, cpad, y)
            v = (a + b) if use_b else a
            ref = np.zeros((n, h, w, cpad), np.float16)
            ref[..., :c] = (v * s).astype(np.float16).transpose(0, 2, 3, 1)
            assert np.array_equal(y.cpu().numpy().view(np.uint16), ref.view(np.uint16)), (use_b, k)
            # unpack channels [c0, c0 + cc) back, plain and accumulating
            x16 = y.cpu().numpy()
            for c0, cc in ((0, c), (cpad - max(1, c // 2), max(1, c // 2))):
                prev = rng.standard_normal((n, cc, h, w)).astype(np.float32)
                for acc in (False, True):
                    out = _t(prev.copy()) if acc else torch.full((n, cc, h, w), float('nan'), device=DEV)
                    ops.grad_unpack(y, cc, sc, c_offset=c0, y=out, accumulate=acc)
                    r = x16[..., c0:c0 + cc].astype(np.float32).transpose(0, 3, 1, 2) * inv
                    if acc:
                        r = prev + r
                    assert np.array_equal(out.cpu().numpy().view(np.uint32), r.astype(np.float32).view(np.uint32)), \
                        (use_b, k, c0, acc)


# ------------------------------------------------------------------------------------------ bias_grad
@pytest.mark.parametrize('c', [8, 24, 48, 64, 128, 256])
def test_bias_grad_sizes_and_guard_band(ops, c):
    import torch
    rows = 256 // (c // 8)
    for npix in (1, 7, rows * 16 - 1, rows * 16 + 1, 1_000_003):
        for c_real in (sorted({c, max(1, c - 5), 1}) if npix < 10 ** 6 else (c,)):
            rng = np.random.default_rng(npix + c + c_real)
            dz = (rng.integers(-64, 64, (npix, c), dtype=np.int8).astype(np.float16) / np.float16(8)).astype(np.float16)
            dz[:, c_real:] = np.float16(1e4)                  # channels past c_real must not reach db
            k = (npix * c) % 7 - 3
            sc, s, inv = _scale_obj(ops, k)
            band = torch.full((c_real + 37,), float('nan'), device=DEV)
            db = band[16:16 + c_real]
            db0 = rng.uniform(-1, 1, c_real).astype(np.float32)
            db.copy_(torch.from_numpy(db0))
            ops.bias_grad(_t(dz.reshape(1, 1, npix, c)), db, sc)
            ref = db0 + dz[:, :c_real].sum(0, dtype=np.float64) * float(inv)
            bound = _gamma(npix + 1) * (np.abs(db0) + np.abs(dz[:, :c_real]).sum(0, dtype=np.float64) * float(inv)) + \
                np.abs(ref) * 2.0 ** -23
            got = db.cpu().numpy().astype(np.float64)
            assert np.all(np.abs(got - ref) <= bound), (npix, c_real, float(np.max(np.abs(got - ref) / bound)))
            g = band.cpu().numpy()
            assert np.isnan(g[:16]).all() and np.isnan(g[16 + c_real:]).all(), (npix, c_real, 'guard band written')


# ------------------------------------------------------------------------------------------ upsample_bwd
def _up_matrix(L, s, bicubic):
    """[s*L, L] float64 matrix of the 1-D upsample, from the oracle applied to basis vectors"""
    from oracle import ops_oracle as K
    eye = np.eye(L, dtype=np.float32).reshape(L, 1, L, 1)
    f = K.bicubic_upsample if bicubic else K.bilinear_upsample
    return f(eye, s)[:, 0, :, 0].T.astype(np.float64)


SIZES = (1, 2, 3, 5, 8, 9, 31, 33)


@pytest.mark.parametrize('s', [2, 4])
@pytest.mark.parametrize('bicubic', [True, False], ids=['bicubic', 'bilinear'])
def test_upsample_bwd_is_the_transposed_upsample(ops, s, bicubic):
    import torch
    mode = 0 if bicubic else 1
    for h in SIZES:
        my = _up_matrix(h, s, bicubic)
        for w in SIZES:
            mx = _up_matrix(w, s, bicubic)
            rng = np.random.default_rng(h * 100 + w + s)
            gy = rng.uniform(-1, 1, (2, 3, s * h, s * w)).astype(np.float32)
            core = np.einsum('Yy,ncYX,Xx->ncyx', my, gy.astype(np.float64), mx)
            acore = np.einsum('Yy,ncYX,Xx->ncyx', np.abs(my), np.abs(gy.astype(np.float64)), np.abs(mx))
            for mul in (1.0, float(s), -0.5):
                for acc in (False, True):
                    prev = rng.uniform(-1, 1, (2, 3, h, w)).astype(np.float32)
                    gx = _t(prev.copy()) if acc else torch.full((2, 3, h, w), float('nan'), device=DEV)
                    ops.upsample_bwd(_t(gy), s, mode, mul=mul, gx=gx, accumulate=acc)
                    ref = mul * core + (prev if acc else 0)
                    bound = _gamma(32 * s + 4) * (abs(mul) * acore + (np.abs(prev) if acc else 0)) + \
                        np.abs(ref) * 2.0 ** -23
                    got = gx.cpu().numpy().astype(np.float64)
                    assert np.all(np.abs(got - ref) <= bound), (h, w, mul, acc, float(np.nanmax(np.abs(got - ref))))


# ------------------------------------------------------------------------------------------ depth_to_space
@pytest.mark.parametrize('s', [2, 4])
def test_depth_to_space_zeroes_the_remainder(ops, s):
    import torch
    L = sys.modules['tecogan-pytorch_b200.lib']
    for h, w in ((s + 1, 2 * s + s - 1), (3 * s + 1, s), (2 * s, 2 * s + 1)):
        n, c = 2, 3
        oh, ow = h // s, w // s
        gy = np.random.default_rng(h * w).standard_normal((n, c * s * s, oh, ow)).astype(np.float32)
        gx = torch.full((n, c, h, w), float('nan'), device=DEV)
        gyt = _t(gy)
        rc = L.load().tg_depth_to_space_nchw_f32(ctypes.c_void_p(gyt.data_ptr()), ctypes.c_void_p(gx.data_ptr()),
                                                 n, c, h, w, s, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        assert rc == 0
        ref = np.zeros((n, c, h, w), np.float32)
        for sy in range(s):
            for sx in range(s):
                ref[:, :, sy:oh * s:s, sx:ow * s:s] = gy[:, (sy * s + sx) * c:(sy * s + sx + 1) * c]
        assert np.array_equal(gx.cpu().numpy(), ref), (h, w)


# ------------------------------------------------------------------------------------------ maxpool2x2_bwd
def _maxpool_bwd_ref(x, gy, act):
    n, h, w, c = x.shape
    gx = np.zeros_like(x)
    slope = {0: None, 1: np.float32(0), 2: np.float32(0.2)}[act]
    for yo in range(h // 2):
        for xo in range(w // 2):
            win = x[:, 2 * yo:2 * yo + 2, 2 * xo:2 * xo + 2].reshape(n, 4, c).astype(np.float32)
            arg = np.argmax(win == win.max(1, keepdims=True), axis=1)      # first maximum, row-major
            xv = np.take_along_axis(win, arg[:, None], 1)[:, 0]
            g = gy[:, yo, xo].astype(np.float32)
            if slope is not None:
                g = np.where(xv > 0, g, g * slope)
            for q in range(4):
                sel = arg == q
                gx[:, 2 * yo + q // 2, 2 * xo + q % 2][sel] = g[sel].astype(np.float16)
    return gx


@pytest.mark.parametrize('c', [8, 64, 256])
@pytest.mark.parametrize('act', [0, 1, 2], ids=['none', 'relu', 'lrelu'])
def test_maxpool2x2_bwd_ties_bit_exact(ops, c, act):
    import torch
    for h, w in ((2, 2), (5, 7), (6, 9), (9, 4)):
        rng = np.random.default_rng(c + act + h * w)
        x = rng.choice(np.array([-1.5, -0.0, 0.0, 0.75, 2.0], np.float16), size=(2, h, w, c))
        gy = rng.uniform(-3, 3, (2, h // 2, w // 2, c)).astype(np.float16)
        gx = torch.full((2, h, w, c), float('nan'), dtype=torch.float16, device=DEV)
        ops.maxpool2x2_bwd(_t(x), _t(gy), act, gx)
        ref = _maxpool_bwd_ref(x, gy, act)
        assert np.array_equal(gx.cpu().numpy().view(np.uint16), ref.view(np.uint16)), (h, w)


# ------------------------------------------------------------------------------------------ upsample2x_bwd
@pytest.mark.parametrize('h,w', [(1, 1), (1, 5), (2, 3), (3, 2), (3, 7), (7, 1), (5, 9)])
def test_upsample2x_bwd_small_and_ragged(ops, h, w):
    import torch
    c = 16
    rng = np.random.default_rng(h * 10 + w)
    gy = rng.uniform(-2, 2, (2, 2 * h, 2 * w, c)).astype(np.float16)
    m = rng.uniform(-1, 1, (2, h, w, c)).astype(np.float16)
    my, mx = _up_matrix(h, 2, False), _up_matrix(w, 2, False)
    g64 = gy.astype(np.float64)
    core = np.einsum('Yy,nYXc,Xx->nyxc', my, g64, mx)
    acore = np.einsum('Yy,nYXc,Xx->nyxc', np.abs(my), np.abs(g64), np.abs(mx))
    for act in (0, 1, 2):
        d = np.ones_like(core) if act == 0 else np.where(m > 0, 1.0, 0.0 if act == 1 else 0.2)
        gx = torch.full((2, h, w, c), float('nan'), dtype=torch.float16, device=DEV)
        ops.upsample2x_bwd(_t(gy), _t(m), act, gx)
        ref = core * d
        ulp16 = np.where(ref == 0, 0.0, 2.0 ** (np.floor(np.log2(np.maximum(np.abs(ref), 2.0 ** -14))) - 10))
        bound = _gamma(18) * acore * d + ulp16
        got = gx.cpu().numpy().astype(np.float64)
        assert np.all(np.abs(got - ref) <= bound), (act, float(np.nanmax(np.abs(got - ref))))
