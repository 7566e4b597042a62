"""CPU tests (no GPU): the plan of a temporally padded stream, FRNet.stream(pad_front=p, padding_mode=...).

PadSchedule is driven exactly as the engine drives it (per push: the caller's resets, then per frame the cuts the
ingest found and every frame that became ready; per flush: the rest, then a restart) and its warm-up / main steps
are run on symbolic state.  For every slot the sequence of (lr_curr, lr_prev, hr_prev) that the steps consume must
be the sequence infer_sequence consumes on pad_sequence(shot)[0] for each of its shots, with exactly the shot's own
frames produced.  pad_sequence is the reference's own BaseModel.pad_sequence where the reference is installed, and
oracle/pad_sequence.py's restatement otherwise."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402
from oracle import pad_sequence as PS          # noqa: E402

E = sys.modules['tecogan-pytorch_b200.engine']
PAD = PS.reference_pad_sequence() or PS.pad_sequence
GARBAGE = 'garbage'                            # warm state of a slot that a warm-up step did not feed


def _padded_ids(first, length, p, mode):
    """Frame ids first .. first+length-1 padded as the reference pads them, and the pad count.  The reference
    asserts q < length in both modes; a 'replicate' pad depends on the first frame only, so a shorter shot is padded
    as a lengthened one and cut back."""
    q = E.pad_count(p, mode, length)
    ids = torch.arange(first, first + max(length, q + 1), dtype=torch.float64).view(-1, 1, 1, 1)
    padded, q2 = PAD(ids, q, mode)
    assert q2 == q
    return [int(v) for v in padded.view(-1)][:q + length], q


def _consumed(seq):
    """infer_sequence over frame ids seq: per step (lr_curr, lr_prev, hr_prev), hr_prev the history of the steps
    before (() = zeros, as frame 0 of the reference's loop)."""
    out, hist, prev = [], (), None
    for f in seq:
        out.append((f, prev, hist))
        hist = hist + ((f, prev),)
        prev = f
    return out


class Sim:
    """PadSchedule driven as PaddedStreamEngine drives it, its steps run on symbolic per-slot state."""

    def __init__(self, n, p, mode):
        self.n, self.p, self.mode = n, p, mode
        self.sched = E.PadSchedule(n, p, mode)
        self.main = [(None, ())] * n          # (lr_prev, hr_prev) of the main state
        self.warm = [(GARBAGE, GARBAGE)] * n
        self.trace = [[] for _ in range(n)]   # per slot: consumed (lr_curr, lr_prev, hr_prev)
        self.produced = []                    # frame ids, in order
        self.rows = []                        # frames returned by each push / flush

    def _produce(self, j, warm, main):
        for step in warm:
            for k, (cur, mode) in enumerate(step):
                if cur is None:
                    self.warm[k] = (GARBAGE, GARBAGE)   # the batch-n step runs on stale state: never to be read
                    continue
                lr, hr = (None, ()) if mode == E.ZERO else self.warm[k]
                assert lr != GARBAGE and hr != GARBAGE
                self.trace[k].append((cur, lr, hr))
                self.warm[k] = (cur, hr + ((cur, lr),))
        for k, (cur, mode, prev) in enumerate(main):
            assert cur == j
            if mode == E.ZERO:
                lr, hr = None, ()
            elif mode == E.LOAD:
                lr, hr = prev, self.warm[k][1]
                assert hr != GARBAGE and self.warm[k][0] == prev, 'lr_prev must be the last warm-up frame'
            else:
                lr, hr = self.main[k]
            self.trace[k].append((cur, lr, hr))
            self.main[k] = (cur, hr + ((cur, lr),))
        self.produced.append(j)

    def push(self, k, resets=(), cuts=None):
        """k frames; `resets` slots start a video at the first; cuts {offset: slots} detected by the ingest."""
        s, rows = self.sched, 0
        s.start(resets)
        for i in range(k):
            s.ingest((cuts or {}).get(i, ()))
            while s.ready():
                self._produce(*s.next())
                rows += 1
        self.rows.append(rows)

    def flush(self):
        s, rows = self.sched, 0
        while s.ready(flush=True):
            self._produce(*s.next(flush=True))
            rows += 1
        s.restart()
        self.rows.append(rows)


def _run(n, p, mode, script):
    """script: ('push', k, resets, {offset: cut slots}) and ('flush',) items; a flush is added at the end.  Returns
    the Sim and, per slot, the shots [(first, length)] the script makes."""
    sim = Sim(n, p, mode)
    starts = [set() for _ in range(n)]
    ends = {0}                                # frames where every slot starts (stream start, after a flush)
    t = 0
    for item in list(script) + [('flush',)]:
        if item[0] == 'push':
            _, k, resets, cuts = item
            resets = sorted(set(resets) | (set(range(n)) if t in ends else set()))
            for r in resets:
                starts[r].add(t)
            for off, slots in (cuts or {}).items():
                for r in slots:
                    starts[r].add(t + off)
            sim.push(k, resets, cuts)
            t += k
        else:
            sim.flush()
            ends.add(t)
    shots = []
    for k in range(n):
        b = sorted(x for x in starts[k] | ends if x < t) + [t]
        shots.append([(a, c - a) for a, c in zip(b[:-1], b[1:]) if c > a])
    return sim, shots, t


def _check(n, p, mode, script):
    sim, shots, total = _run(n, p, mode, script)
    assert sim.produced == list(range(total)), 'every frame once, in order'
    for k in range(n):
        want = []
        for first, length in shots[k]:
            seq, q = _padded_ids(first, length, p, mode)
            assert seq[q:] == list(range(first, first + length))
            want += _consumed(seq)
        assert sim.trace[k] == want, (k, shots[k])
    return sim


PS_ = [0, 1, 2, 5]
MODES = ['reflect', 'replicate']


@pytest.mark.parametrize('p', PS_)
@pytest.mark.parametrize('mode', MODES)
def test_shots_of_every_short_length(p, mode):
    """One slot, shots of 1 .. p+2 frames back to back (cuts on consecutive frames where the length is 1), in
    pushes of 1 .. 7 frames."""
    for push in range(1, 8):
        lengths = list(range(1, p + 3)) + [1, 1, 2, 1]
        cut_frames, t = set(), 0
        for length in lengths:
            cut_frames.add(t)
            t += length
        script, f = [], 0
        while f < t:
            k = min(push, t - f)
            script.append(('push', k, (), {i: [0] for i in range(k) if f + i in cut_frames and f + i > 0}))
            f += k
        _check(1, p, mode, script)


@pytest.mark.parametrize('p', PS_)
@pytest.mark.parametrize('mode', MODES)
def test_three_slots_with_cuts_and_resets_at_push_edges(p, mode):
    """Three slots with different shot patterns: cuts on the first and the last frame of a push, a reset of one slot
    in a push (its previous video ends with the previous push), resets of two slots at once, one-frame pushes."""
    script = [
        ('push', 4, (), {0: [], 3: [1]}),                 # slot 1 cut on the last frame
        ('push', 3, [2], {0: [0]}),                       # slot 2 reset, slot 0 cut on the first frame
        ('push', 1, [0], {0: [1]}),                       # one-frame push: reset and cut on it
        ('push', 7, (), {1: [0, 2], 2: [0], 6: [1]}),
        ('push', 2, [0, 1], {1: [2]}),
        ('push', 5, (), {}),
    ]
    sim = _check(3, p, mode, script)
    lag = p if mode == 'reflect' else 0
    assert sim.rows[0] == max(0, 4 - lag)
    assert sum(sim.rows) == 22 and sim.rows[-1] == min(lag, 22)


@pytest.mark.parametrize('p', PS_)
@pytest.mark.parametrize('mode', MODES)
@pytest.mark.parametrize('push', [1, 2, 3, 7])
def test_flush_returns_the_held_frames(p, mode, push):
    """Streams of 0 .. p+3 frames, then flush: the flush returns min(lag, frames) frames, and a second video after it
    starts fresh in every slot (and is flushed in turn)."""
    lag = p if mode == 'reflect' else 0
    for total in range(0, p + 4):
        script, f = [], 0
        while f < total:
            k = min(push, total - f)
            script.append(('push', k, (), {}))
            f += k
        script += [('flush',), ('push', 3, (), {1: [1]}), ('push', 2, [0], {})]
        sim = _check(2, p, mode, script)
        flushed = sim.rows[len(script) - 3]
        assert flushed == min(lag, total)
        assert sim.rows[-1] == min(lag, 5)


@pytest.mark.parametrize('p', PS_)
@pytest.mark.parametrize('mode', MODES)
def test_random_scripts(p, mode):
    rng = np.random.default_rng(100 * p + len(mode))
    for _ in range(30):
        n = int(rng.integers(1, 4))
        script = []
        for _ in range(int(rng.integers(1, 8))):
            if rng.random() < 0.15:
                script.append(('flush',))
                continue
            k = int(rng.integers(1, 8))
            resets = [s for s in range(n) if rng.random() < 0.2]
            cuts = {i: [s for s in range(n) if rng.random() < 0.25] for i in range(k)}
            script.append(('push', k, resets, cuts))
        _check(n, p, mode, script)


def test_warm_up_is_shared_and_ends_on_the_last_step():
    """Slots starting a shot at the same frame share the warm-up steps; each slot's run ends on the last one."""
    warm, main = E.plan_step(10, [6, None, 3, 1], 5, 'reflect')     # q = 5, -, 2, 0
    assert len(warm) == 5
    assert [s[0] for s in warm] == [(15, E.ZERO), (14, E.KEEP), (13, E.KEEP), (12, E.KEEP), (11, E.KEEP)]
    assert [s[2] for s in warm] == [(None, E.KEEP)] * 3 + [(12, E.ZERO), (11, E.KEEP)]
    assert all(s[1] == (None, E.KEEP) and s[3] == (None, E.KEEP) for s in warm)
    assert main == [(10, E.LOAD, 11), (10, E.KEEP, None), (10, E.LOAD, 11), (10, E.ZERO, None)]
    warm, main = E.plan_step(4, [None, 1], 3, 'replicate')
    assert [s[1] for s in warm] == [(4, E.ZERO), (4, E.KEEP), (4, E.KEEP)] and main[1] == (4, E.LOAD, 4)


def test_plan_matches_schedule():
    """plan() (the whole schedule from shot starts) is what PadSchedule produces frame by frame."""
    starts = [{3, 4, 9}, {1}, set()]
    whole = E.plan(starts, 12, 5, 'reflect')
    sim = Sim(3, 5, 'reflect')
    got = []
    sim._produce = lambda j, w, m: got.append((w, m))
    sim.push(12, [0, 1, 2], {i: [k for k in range(3) if i in starts[k]] for i in range(12)})
    sim.flush()
    assert got == whole


def _net():
    return T.FRNet(3, 3, 64, 2, 'BD', 4).eval()


@pytest.mark.parametrize('bad', [-1, 33, 2.0, '5', True, None])
def test_pad_front_is_validated(bad):
    with pytest.raises(ValueError, match='pad_front'):
        _net().stream(2, 16, 24, device='cuda', pad_front=bad)


@pytest.mark.parametrize('bad', ['zero', 'Reflect', None, 1])
def test_padding_mode_is_validated(bad):
    with pytest.raises(ValueError, match='padding_mode'):
        _net().stream(2, 16, 24, device='cuda', pad_front=2, padding_mode=bad)


@pytest.mark.parametrize('p', [0, 1, 32])
def test_valid_padding_opens_a_stream_without_a_device(p):
    s = _net().stream(2, 16, 24, device='cuda', pad_front=p, padding_mode='replicate')
    assert s.pad_front == p and s.padding_mode == 'replicate'


def test_restatement_matches_the_reference_pad_sequence():
    ref = PS.reference_pad_sequence()
    if ref is None:
        pytest.skip('the reference is not installed (oracle/_ref)')
    x = torch.arange(7, dtype=torch.float32).view(7, 1, 1, 1).expand(7, 2, 3, 4).contiguous()
    for mode in MODES:
        for q in range(7):
            a, qa = ref(x, q, mode)
            b, qb = PS.pad_sequence(x, q, mode)
            assert qa == qb == q and torch.equal(a, b)
