"""pytest -m gpu: temporally padded streams, FRNet.stream(pad_front=p, padding_mode=...).

tg_stream_gather is replayed against its contract (oracle/pad_sequence.py gather) with a 0xAB guard band around every
output.  End to end, every frame a padded stream returns is byte-identical to the library's own infer_sequence over
the reference-padded shot it belongs to (pad_sequence(shot, q)[0], outputs [q:]), with shots started by the stream
start, caller resets and detected scene cuts; the cut reports equal those of the unpadded stream."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
import synthetic                               # noqa: E402
from oracle import pad_sequence as PS          # noqa: E402
from oracle import scene_cut as S              # noqa: E402
from oracle import yuv_color as C              # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
E = sys.modules['tecogan-pytorch_b200.engine']
DEV = torch.device('cuda', 0)
BD4 = dict(scale=4, degradation='BD', h=134, w=320)
BI2 = dict(scale=2, degradation='BI', h=36, w=52)
THR = 10.0
G = 37                                         # guard floats around every output (an odd count: misaligned starts)


# ---------------------------------------------------------------------------- the kernel against its contract
def _guarded(shape, fill, offset):
    """A float32 view of `shape` at `offset` floats into a 0xAB-filled buffer with G guard floats after it."""
    size = int(np.prod(shape))
    buf = torch.full((offset + size + G,), 0, dtype=torch.int32, device=DEV)
    buf.view(torch.uint8).fill_(0xAB)
    v = buf.view(torch.float32)[offset:offset + size].view(shape)
    if fill is not None:
        v.copy_(torch.from_numpy(fill))
    return buf, v


@pytest.mark.parametrize('n,c,h,w,s', [(1, 1, 1, 1, 2), (3, 3, 5, 7, 4), (2, 3, 17, 33, 2), (4, 3, 134, 320, 4)])
@pytest.mark.parametrize('offset', [G, G + 1, G + 3], ids=['aligned16', 'off4', 'off12'])
def test_gather_matches_contract(n, c, h, w, s, offset):
    rng = np.random.default_rng(n * 100 + h + offset)
    depth = 4
    ring = torch.from_numpy(rng.uniform(-1, 2, (depth, n, c, h, w)).astype(np.float32)).to(DEV)
    warm = torch.from_numpy(rng.uniform(-1, 2, (n, c, s * h, s * w)).astype(np.float32)).to(DEV)
    for trial in range(6):
        lr0 = rng.uniform(-1, 2, (n, c, h, w)).astype(np.float32)
        prev0 = rng.uniform(-1, 2, (n, c, h, w)).astype(np.float32)
        hr0 = rng.uniform(-1, 2, (n, c, s * h, s * w)).astype(np.float32)
        cur = rng.integers(-2, depth + 2, n)
        mode = rng.integers(0, 4, n)                      # 3: not a mode, kept
        prev = rng.integers(-1, depth + 1, n)
        table = np.concatenate([cur, mode, prev]).astype(np.int32)
        bufs = [_guarded(x.shape, x, offset - (i if trial % 2 else 0)) for i, x in enumerate((lr0, prev0, hr0))]
        (lb, lv), (pb, pv), (hb, hv) = bufs
        wh = None if trial == 5 else warm
        ops.stream_gather(ring, torch.from_numpy(table).to(DEV), wh, lv, pv, hv, s)
        torch.cuda.synchronize()
        want = [lr0.copy(), prev0.copy(), hr0.copy()]
        PS.gather(ring.cpu().numpy(), table, None if wh is None else wh.cpu().numpy(), *want)
        for (buf, v), x, off in zip(bufs, want, [offset - (i if trial % 2 else 0) for i in range(3)]):
            assert np.array_equal(v.cpu().numpy().view(np.int32), x.view(np.int32)), (trial, table)
            raw = buf.view(torch.uint8).cpu().numpy()
            assert (raw[:4 * off] == 0xAB).all() and (raw[4 * (off + x.size):] == 0xAB).all(), 'guard band written'


def test_gather_rejects_bad_arguments():
    ring = torch.zeros(3, 2, 3, 4, 5, device=DEV)
    lr = torch.zeros(2, 3, 4, 5, device=DEV)
    hr = torch.zeros(2, 3, 16, 20, device=DEV)
    tab = torch.zeros(6, dtype=torch.int32, device=DEV)
    with pytest.raises(T.TecoganB200Error):
        ops.stream_gather(ring, tab[:5], None, lr, lr.clone(), hr, 4)
    with pytest.raises(T.TecoganB200Error):
        ops.stream_gather(ring, tab, None, lr, lr.clone(), hr, 2)
    with pytest.raises(T.TecoganB200Error, match='scale 3'):
        ops.stream_gather(ring, tab, None, lr, lr.clone(), torch.zeros(2, 3, 12, 15, device=DEV), 3)


# ---------------------------------------------------------------------------- streams end to end
def _net(scale, degradation):
    net = T.FRNet(3, 3, 64, 10, degradation, scale)
    net.load_state_dict(synthetic.make_frnet_params(0, scale=scale, degradation=degradation, gain=1.0), strict=True)
    return net.to(DEV).eval()


@pytest.fixture(scope='module')
def nets():
    return {'bd4': _net(4, 'BD'), 'bi2': _net(2, 'BI')}


def _u8(clip):
    """fp32 [t,3,h,w] in [0,1] -> uint8 [t,h,w,3]"""
    return np.rint(clip.numpy() * 255.0).astype(np.uint8).transpose(0, 2, 3, 1)


def _clips(h, w):
    """uint8 RGB [3,18,h,w,3]: slot 0 two shots of 9 frames (a cut at 9); slot 1 one clip (the test resets it);
    slot 2 shots of 3, 2 and 13 frames (cuts at 3 and 5: shots shorter than p + 1)."""
    mk = lambda seed, t: _u8(synthetic.make_clip(seed, t, 3, h, w))             # noqa: E731
    s0 = np.concatenate([mk(1, 9), mk(2, 9)])
    s1 = mk(3, 18)
    s2 = np.concatenate([mk(4, 3), mk(5, 2), mk(6, 13)])
    return np.ascontiguousarray(np.stack([s0, s1, s2]))


def _f32(u8):
    return u8.astype(np.float32) / np.float32(255)


def _padded_ids(first, length, p, mode):
    q = E.pad_count(p, mode, length)
    ids = torch.arange(first, first + max(length, q + 1), dtype=torch.float64).view(-1, 1, 1, 1)
    padded, _ = PS.pad_sequence(ids, q, mode)
    return [int(v) for v in padded.view(-1)][:q + length], q


def _expected(net, dec, starts, p, mode):
    """dec fp32 [n,T,h,w,3] decoded LR frames, starts per slot the shot starts -> uint8 [n,T,H,W,3]: per shot,
    infer_sequence over the padded shot (placed in every slot of a batch of n, so slot k is computed where the stream
    computes it), outputs [q:]."""
    n, t = dec.shape[:2]
    out = None
    for k in range(n):
        b = sorted(set(starts[k]) | {0}) + [t]
        for a, e in zip(b[:-1], b[1:]):
            ids, q = _padded_ids(a, e - a, p, mode)
            seq = np.ascontiguousarray(dec[k, ids].transpose(0, 3, 1, 2))           # tchw
            batch = torch.from_numpy(np.ascontiguousarray(np.broadcast_to(seq, (n, *seq.shape))))
            res = net.infer_sequence(batch, DEV)[k, q:]
            if out is None:
                out = np.empty((n, t, *res.shape[1:]), np.uint8)
            out[k, a:e] = res
    return out


def _drive(stream, frames, chunks, resets, out='host'):
    """Push frames [n,T,...] in chunks (resets: {push index: slots}), then flush.  -> (frames, cuts, scores, rows)"""
    res, cuts, scores, rows, i = [], [], [], [], 0
    for j, k in enumerate(chunks):
        src = torch.from_numpy(np.ascontiguousarray(frames[:, i:i + k]))
        r = [s in resets.get(j, ()) for s in range(stream.n)]
        o = stream.push(src.to(DEV) if out == 'device' else src, reset=r, out=out)
        res.append(o.cpu().numpy() if out == 'device' else o)
        rows.append(res[-1].shape[1])
        if stream.scene_cut is not None:
            lc, ls = stream.last_cuts, stream.last_scores
            if out == 'device':
                lc, ls = lc.cpu().numpy(), ls.cpu().numpy()
            assert lc.shape == ls.shape == (stream.n, rows[-1])
            cuts.append(lc)
            scores.append(ls)
        i += k
    o = stream.flush(out=out)
    res.append(o.cpu().numpy() if out == 'device' else o)
    rows.append(res[-1].shape[1])
    if stream.scene_cut is not None:
        lc, ls = stream.last_cuts, stream.last_scores
        cuts.append(lc.cpu().numpy() if out == 'device' else lc)
        scores.append(ls.cpu().numpy() if out == 'device' else ls)
    cat = lambda v: np.concatenate(v, axis=1) if v else None                   # noqa: E731
    return cat(res), cat(cuts), cat(scores), rows


def _reset_push(chunks, frame):
    """Index of the first push that starts at or after `frame`."""
    f = 0
    for j, k in enumerate(chunks):
        if f >= frame:
            return j
        f += k
    return len(chunks)


_EXPECTED = {}

CASES = [('bd4', 'reflect', 5, c) for c in (1, 4, 7)] + [('bd4', 'replicate', 3, 4), ('bi2', 'reflect', 5, 4),
                                                           ('bi2', 'replicate', 3, 7), ('bi2', 'reflect', 5, 1)]


@pytest.mark.parametrize('geom,mode,p,push', CASES)
def test_padded_stream_matches_padded_infer_sequence(geom, mode, p, push, nets):
    """n = 3, 18 frames, scene_cut=10: slot 0 cuts at 9, slot 1 is reset by the caller in mid-stream, slot 2 has
    shots of 3 and 2 frames; pushes of `push` frames, then flush."""
    net, g = nets[geom], (BD4 if geom == 'bd4' else BI2)
    rgb = _clips(g['h'], g['w'])
    n, t = rgb.shape[:2]
    chunks = [push] * (t // push) + ([t % push] if t % push else [])
    rp = _reset_push(chunks, 7)
    reset_at = sum(chunks[:rp])
    dec = _f32(rgb)
    o_cuts = np.stack([S.stream(dec[k], {reset_at} if k == 1 else set(), THR)[1] for k in range(n)])
    assert o_cuts[0, 9] and o_cuts[2, 3] and o_cuts[2, 5], np.nonzero(o_cuts)
    starts = [set(np.flatnonzero(o_cuts[k])) for k in range(n)]
    starts[1].add(reset_at)
    key = (geom, mode, p, reset_at)
    if key not in _EXPECTED:
        _EXPECTED[key] = _expected(net, dec, starts, p, mode)
    want = _EXPECTED[key]
    s = net.stream(n, g['h'], g['w'], device=DEV, scene_cut=THR, pad_front=p, padding_mode=mode)
    got, cuts, scores, rows = _drive(s, rgb, chunks, {rp: [1]})
    s.close()
    lag = p if mode == 'reflect' else 0
    emitted = np.cumsum(chunks)
    assert rows[:-1] == [int(min(e, max(0, e - lag)) - max(0, e - k - lag)) for e, k in zip(emitted, chunks)]
    assert rows[-1] == lag
    assert got.shape == want.shape and np.array_equal(got, want), int((got != want).sum())
    # the reports are the unpadded stream's, frame for frame
    plain = net.stream(n, g['h'], g['w'], device=DEV, scene_cut=THR)
    _, pc, psc, _ = _drive(plain, rgb, chunks, {rp: [1]})
    plain.close()
    assert np.array_equal(cuts, pc) and np.array_equal(scores.view(np.int64), psc.view(np.int64))


def _workaround(net, frames, dec_shape, shots, p, mode, kw, out='host'):
    """The bytes of a padded stream whose every slot has the same shots, made with an unpadded stream: each shot's
    pad frames pushed in front of it with a reset of every slot, those outputs dropped."""
    n = frames.shape[0]
    s = net.stream(n, *dec_shape, device=DEV, **kw)
    res = []
    for a, length in shots:
        ids, q = _padded_ids(a, length, p, mode)
        o = s.push(torch.from_numpy(np.ascontiguousarray(frames[:, ids])), reset=[True] * n)
        res.append(o[:, q:])
    s.close()
    return np.concatenate(res, axis=1)


FORMATS = {
    'nv12_in': lambda rgb: (dict(input='nv12'), C.rgb_to_yuv(rgb, 'nv12', 'bt601')),
    'p010_out': lambda rgb: (dict(out_format='p010', out_color='bt709'), rgb),
    'out_size': lambda rgb: (dict(out_size=(54, 130)), rgb),
    'crop_out_frame': lambda rgb: (dict(crop=(4, 6, 28, 40), out_frame=(64, 96)), rgb),
}


@pytest.mark.parametrize('fmt', list(FORMATS) + ['device'])
def test_padded_stream_composes_with_formats(fmt, nets):
    """bi2, reflect p = 3, n = 3 slots sharing their shots (a reset of every slot at frame 7): each format gives the
    bytes of the unpadded stream of that format fed the padded shots."""
    net, g = nets['bi2'], BI2
    rgb = _clips(g['h'], g['w'])[:, :12]
    kw, frames = FORMATS.get(fmt, lambda r: (dict(), r))(rgb)
    p, mode = 3, 'reflect'
    shots = [(0, 7), (7, 5)]
    want = _workaround(net, frames, (g['h'], g['w']), shots, p, mode, kw)
    out = 'device' if fmt == 'device' else 'host'
    s = net.stream(3, g['h'], g['w'], device=DEV, pad_front=p, padding_mode=mode, **kw)
    got, _, _, _ = _drive(s, frames, [4, 3, 5], {2: [0, 1, 2]}, out=out)
    s.close()
    assert got.dtype == want.dtype and np.array_equal(got, want), (fmt, int((got != want).sum()))


def test_benchmark_shape_reflect_5(nets):
    import bench
    bench.select_workload('bd4')
    n, (c, h, w) = bench.CLIPS_PER_GPU, bench.LR
    clips = bench.synthetic_clips(n, 24, seed=100)                          # [n,24,c,h,w] fp32
    u8 = np.ascontiguousarray(np.rint(clips.numpy() * 255.0).astype(np.uint8).transpose(0, 1, 3, 4, 2))
    dec = _f32(u8)
    want = _expected(nets['bd4'], dec, [set()] * n, 5, 'reflect')
    s = nets['bd4'].stream(n, h, w, device=DEV, pad_front=5)
    got, _, _, rows = _drive(s, u8, [16, 8], {})
    s.close()
    assert rows == [11, 8, 5]
    assert np.array_equal(got, want), int((got != want).sum())


def test_pad_front_0_is_the_plain_stream(nets):
    net, g = nets['bd4'], BD4
    rgb = _clips(g['h'], g['w'])[:, :6]
    a = net.stream(3, g['h'], g['w'], device=DEV)
    b = net.stream(3, g['h'], g['w'], device=DEV, pad_front=0, padding_mode='replicate')
    wa, wb = a.push(rgb), b.push(rgb)
    assert type(b._engine) is E.StreamEngine
    assert a._engine.launches_per_step == b._engine.launches_per_step
    assert np.array_equal(wa, wb)
    assert b.flush().shape == (3, 0, 4 * g['h'], 4 * g['w'], 3)
    a.close()
    b.close()


def test_single_channel_stream_with_scene_cut_and_padding():
    """FRNet(1, 1) at 2x BI, n = 3 slots of single-channel frames (channel 0 of the RGB clips: cuts at 9, 3 and 5),
    scene_cut=10, reflect p = 3, pushes of 4: frames [n,k,h,w,1] in, the bytes of infer_sequence over each padded shot
    out, and the cuts the oracle finds"""
    g, p, mode, n = BI2, 3, 'reflect', 3
    net = T.FRNet(1, 1, 64, 10, 'BI', 2)
    net.load_state_dict(synthetic.make_frnet_params(0, in_nc=1, out_nc=1, scale=2, degradation='BI', gain=1.0),
                        strict=True)
    net = net.to(DEV).eval()
    gray = np.ascontiguousarray(_clips(g['h'], g['w'])[..., :1])
    t = gray.shape[1]
    dec = _f32(gray)
    o_cuts = np.stack([S.stream(dec[k].transpose(0, 3, 1, 2), set(), THR)[1] for k in range(n)])
    assert o_cuts[0, 9] and o_cuts[2, 3] and o_cuts[2, 5], np.nonzero(o_cuts)
    want = _expected(net, dec, [set(np.flatnonzero(o_cuts[k])) for k in range(n)], p, mode)
    s = net.stream(n, g['h'], g['w'], device=DEV, scene_cut=THR, pad_front=p, padding_mode=mode)
    got, cuts, _, _ = _drive(s, gray, [4] * (t // 4) + [t % 4], {})
    s.close()
    assert got.shape == (n, t, 2 * g['h'], 2 * g['w'], 1) and np.array_equal(got, want), int((got != want).sum())
    assert np.array_equal(cuts, o_cuts)
