"""pytest -m gpu: the launch plan of a stream -- every ops call a stream's engine makes while it is built (the fills
of out_frame's bars, the warm-up and capture of each graph) and while it runs a push of 3 frames (a padded stream's
ingest), in order, with the engine buffer each tensor argument points at and every other argument as passed.

The byte tests (test_stream*_gpu.py, test_scene_cut_gpu.py) show that a stream computes the right frames and the
launch-count tests that it makes the right number of launches; this one pins which launches, on which buffers, so a
change to how the engine chooses its launches cannot reorder or re-route them unseen.  The net's step_into is one
entry, step_into(lr_curr, lr_prev, hr_prev, out, out_u8); the calls inside it are not listed."""
import inspect
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tecogan_b200 as T                       # noqa: E402

pytestmark = pytest.mark.gpu

ops = sys.modules['tecogan-pytorch_b200.ops']
DEV = torch.device('cuda', 0)
N, H, W = 2, 16, 24
RECORDED = ('stream_frame_in', 'stream_frame_in_yuv420', 'stream_frame_in_yuv', 'stream_frame_in_resample',
            'stream_gather', 'scene_cut', 'resample', 'float_to_uint8_nhwc', 'float_to_uint8_nhwc_window',
            'rgb_u8_to_yuv420', 'rgb_to_yuv', 'fill_black')
# engine buffers; a tensor is named after the buffer of its address and shape, else as a row (and byte offset) of the
# buffer it lies in: score[p] is the float64 view of rep[p]'s first 2n words, ring[r] a row of the ring
BUFFERS = ('inp', 'stage', 'lr', 'hr', 'u8', 'rs', 'yuv', 'pad', 'mask', 'score', 'cut', 'rep', 'prev_mafd', 'work',
           'tables', 'in_tables', 'ring', 'wlr', 'whr', 'mtab', 'wtab', 'rep_ring', 'in_mask')


class Plan:
    """Records the top-level calls of RECORDED and of net.step_into; tensors are named after the push."""

    def __init__(self, net, monkeypatch):
        self.calls, self.depth = [], 0
        for name in RECORDED:
            monkeypatch.setattr(ops, name, self._wrap(name, getattr(ops, name)))
        monkeypatch.setattr(net, 'step_into', self._wrap('step_into', net.step_into))

    def _wrap(self, name, real):
        sig = inspect.signature(real)

        def wrapped(*a, **k):
            if self.depth == 0:
                bound = sig.bind(*a, **k)
                bound.apply_defaults()
                self.calls.append((name, list(bound.arguments.values())))
            self.depth += 1
            try:
                return real(*a, **k)
            finally:
                self.depth -= 1
        return wrapped

    def lines(self, engine):
        leaves = []

        def walk(name, v):
            if isinstance(v, torch.Tensor):
                leaves.append((name, v))
            elif isinstance(v, (list, tuple)):
                for i, x in enumerate(v):
                    walk(f'{name}[{i}]', x)
        for name in BUFFERS:
            walk(name, getattr(engine, name, None))

        def tensor_name(t):
            ptr = t.data_ptr()
            for name, b in leaves:
                if b.data_ptr() == ptr and b.shape == t.shape:
                    return name
            for name, b in leaves:       # a view into a buffer: its row, and the byte offset within the row
                off = ptr - b.data_ptr()
                if b.dim() > 1 and 0 <= off < b.numel() * b.element_size():
                    row = b[0].numel() * b.element_size()
                    return f'{name}[{off // row}]' + (f'+{off % row}' if off % row else '')
            return f'tensor{tuple(t.shape)}'

        def fmt(v):
            if isinstance(v, torch.Tensor):
                return tensor_name(v)
            if isinstance(v, (list, tuple)):
                return '(' + ', '.join(fmt(x) for x in v) + ')'
            return repr(v)
        return [f'{name}({", ".join(fmt(v) for v in args)})' for name, args in self.calls]


def _frames(input, h, w, k=3):
    if input == 'uint8':
        return np.zeros((N, k, h, w, 3), np.uint8)
    if input == 'float32':
        return np.zeros((N, k, 3, h, w), np.float32)
    return np.zeros((N, k, *ops.yuv_frame_shape(input, h, w)), np.uint16 if ops.yuv_depth(input) == 10 else np.uint8)


def launch_plan(net, monkeypatch, h=H, w=W, **kw):
    """The plan lines of a new stream's first push of 3 frames."""
    s = net.stream(N, h, w, device=DEV, **kw)
    plan = Plan(net, monkeypatch)
    s.push(_frames(kw.get('input', 'uint8'), h, w))
    torch.cuda.synchronize()
    lines = plan.lines(s._engine)
    s.close()
    return lines


# (id, stream arguments): h, w are the pushed frames' size (16 x 24 when not given)
CASES = [
    ('u8', {}),
    ('u8_bgr', dict(channel_order='bgr')),
    ('f32', dict(input='float32')),
    ('nv12', dict(input='nv12')),
    ('i420', dict(input='i420')),
    ('nv12_709', dict(input='nv12', in_color='bt709')),
    ('p010', dict(input='p010')),
    ('yuy2', dict(input='yuy2')),
    ('i444_10', dict(input='i444_10')),
    ('out_nv12', dict(out_format='nv12')),
    ('out_nv12_709', dict(out_format='nv12', out_color='bt709')),
    ('out_p010', dict(out_format='p010')),
    ('out_uyvy', dict(out_format='uyvy')),
    ('out_size', dict(out_size=(48, 72))),
    ('out_size_p010', dict(out_size=(48, 72), out_format='p010')),
    ('out_size_nv12', dict(out_size=(48, 72), out_format='nv12')),
    ('crop', dict(h=20, w=28, crop=(2, 2, 16, 24))),
    ('crop_bgr', dict(h=20, w=28, crop=(2, 2, 16, 24), channel_order='bgr')),
    ('crop_nv12', dict(h=20, w=28, crop=(2, 2, 16, 24), input='nv12')),
    ('out_frame', dict(out_frame=(72, 104))),
    ('out_frame_nv12', dict(out_frame=(72, 104), out_format='nv12')),
    ('out_frame_p010', dict(out_frame=(72, 104), out_format='p010')),
    ('out_frame_size', dict(out_frame=(64, 96), out_size=(48, 72))),
    ('out_frame_size_p010', dict(out_frame=(64, 96), out_size=(48, 72), out_format='p010')),
    ('in_size', dict(h=32, w=48, in_size=(16, 24))),
    ('in_size_nv12', dict(h=32, w=48, in_size=(16, 24), input='nv12', scene_cut=10.0)),
    ('in_size_crop', dict(h=36, w=52, crop=(2, 2, 32, 48), in_size=(16, 24))),
    ('scene_cut', dict(scene_cut=10.0)),
    ('scene_cut_nv12_out_size', dict(scene_cut=10.0, input='nv12', out_size=(48, 72), out_format='nv12')),
    ('pad_reflect', dict(pad_front=2)),
    ('pad_replicate', dict(pad_front=2, padding_mode='replicate')),
    ('pad_reflect_cut', dict(pad_front=2, scene_cut=10.0)),
    ('pad_replicate_cut', dict(pad_front=2, padding_mode='replicate', scene_cut=10.0)),
    ('pad_f32_cut', dict(pad_front=2, input='float32', scene_cut=10.0)),
    ('pad_nv12_crop_p010', dict(pad_front=2, h=20, w=28, crop=(2, 2, 16, 24), input='nv12', out_format='p010')),
    ('pad_in_size_out_frame', dict(pad_front=2, h=32, w=48, in_size=(16, 24), out_frame=(72, 104))),
]

EXPECTED = {'u8': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
        'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
        'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
        'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
        'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
        'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
        'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
        'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'u8_bgr': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, True, None)',
            'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
            'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, True, None)',
            'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
            'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, True, None)',
            'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
            'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, True, None)',
            'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'f32': ['stream_frame_in(None, mask[0], lr[0], lr[1], hr[1], 4, False, None)',
         'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
         'stream_frame_in(None, mask[1], lr[1], lr[0], hr[0], 4, False, None)',
         'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
         'stream_frame_in(None, mask[0], lr[0], lr[1], hr[1], 4, False, None)',
         'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
         'stream_frame_in(None, mask[1], lr[1], lr[0], hr[0], 4, False, None)',
         'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'nv12': ["stream_frame_in_yuv420(inp[0], 'nv12', mask[0], lr[0], lr[1], hr[1], 4)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv420(inp[1], 'nv12', mask[1], lr[1], lr[0], hr[0], 4)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
          "stream_frame_in_yuv420(inp[0], 'nv12', mask[0], lr[0], lr[1], hr[1], 4)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv420(inp[1], 'nv12', mask[1], lr[1], lr[0], hr[0], 4)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'i420': ["stream_frame_in_yuv420(inp[0], 'i420', mask[0], lr[0], lr[1], hr[1], 4)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv420(inp[1], 'i420', mask[1], lr[1], lr[0], hr[0], 4)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
          "stream_frame_in_yuv420(inp[0], 'i420', mask[0], lr[0], lr[1], hr[1], 4)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv420(inp[1], 'i420', mask[1], lr[1], lr[0], hr[0], 4)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'nv12_709': ["stream_frame_in_yuv(inp[0], 'nv12', 'bt709', mask[0], lr[0], lr[1], hr[1], 4, None)",
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "stream_frame_in_yuv(inp[1], 'nv12', 'bt709', mask[1], lr[1], lr[0], hr[0], 4, None)",
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "stream_frame_in_yuv(inp[0], 'nv12', 'bt709', mask[0], lr[0], lr[1], hr[1], 4, None)",
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "stream_frame_in_yuv(inp[1], 'nv12', 'bt709', mask[1], lr[1], lr[0], hr[0], 4, None)",
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'p010': ["stream_frame_in_yuv(inp[0], 'p010', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, None)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv(inp[1], 'p010', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, None)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
          "stream_frame_in_yuv(inp[0], 'p010', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, None)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv(inp[1], 'p010', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, None)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'yuy2': ["stream_frame_in_yuv(inp[0], 'yuy2', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, None)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv(inp[1], 'yuy2', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, None)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
          "stream_frame_in_yuv(inp[0], 'yuy2', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, None)",
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          "stream_frame_in_yuv(inp[1], 'yuy2', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, None)",
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'i444_10': ["stream_frame_in_yuv(inp[0], 'i444_10', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, None)",
             'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
             "stream_frame_in_yuv(inp[1], 'i444_10', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, None)",
             'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
             "stream_frame_in_yuv(inp[0], 'i444_10', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, None)",
             'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
             "stream_frame_in_yuv(inp[1], 'i444_10', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, None)",
             'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'out_nv12': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "rgb_u8_to_yuv420(u8[0], 'nv12', yuv[0])",
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "rgb_u8_to_yuv420(u8[1], 'nv12', yuv[1])",
              'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "rgb_u8_to_yuv420(u8[0], 'nv12', yuv[0])",
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "rgb_u8_to_yuv420(u8[1], 'nv12', yuv[1])"],
 'out_nv12_709': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                  'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                  "rgb_to_yuv('nv12', 'bt709', u8[0], None, yuv[0], None)",
                  'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                  'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                  "rgb_to_yuv('nv12', 'bt709', u8[1], None, yuv[1], None)",
                  'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                  'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                  "rgb_to_yuv('nv12', 'bt709', u8[0], None, yuv[0], None)",
                  'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                  'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                  "rgb_to_yuv('nv12', 'bt709', u8[1], None, yuv[1], None)"],
 'out_p010': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "rgb_to_yuv('p010', 'bt601', None, hr[0], yuv[0], None)",
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "rgb_to_yuv('p010', 'bt601', None, hr[1], yuv[1], None)",
              'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "rgb_to_yuv('p010', 'bt601', None, hr[0], yuv[0], None)",
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "rgb_to_yuv('p010', 'bt601', None, hr[1], yuv[1], None)"],
 'out_uyvy': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "rgb_to_yuv('uyvy', 'bt601', u8[0], None, yuv[0], None)",
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "rgb_to_yuv('uyvy', 'bt601', u8[1], None, yuv[1], None)",
              'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              "rgb_to_yuv('uyvy', 'bt601', u8[0], None, yuv[0], None)",
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              "rgb_to_yuv('uyvy', 'bt601', u8[1], None, yuv[1], None)"],
 'out_size': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], None)',
              'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[0], None, None)',
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], None)',
              'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[1], None, None)',
              'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
              'step_into(lr[0], lr[1], hr[1], hr[0], None)',
              'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[0], None, None)',
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
              'step_into(lr[1], lr[0], hr[0], hr[1], None)',
              'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[1], None, None)'],
 'out_size_p010': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                   'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                   'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[0], None)',
                   "rgb_to_yuv('p010', 'bt601', None, rs[0], yuv[0], None)",
                   'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                   'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                   'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[1], None)',
                   "rgb_to_yuv('p010', 'bt601', None, rs[1], yuv[1], None)",
                   'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                   'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                   'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[0], None)',
                   "rgb_to_yuv('p010', 'bt601', None, rs[0], yuv[0], None)",
                   'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                   'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                   'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[1], None)',
                   "rgb_to_yuv('p010', 'bt601', None, rs[1], yuv[1], None)"],
 'out_size_nv12': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                   'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                   'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[0], None, None)',
                   "rgb_u8_to_yuv420(rs[0], 'nv12', yuv[0])",
                   'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                   'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                   'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[1], None, None)',
                   "rgb_u8_to_yuv420(rs[1], 'nv12', yuv[1])",
                   'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                   'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                   'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[0], None, None)',
                   "rgb_u8_to_yuv420(rs[0], 'nv12', yuv[0])",
                   'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                   'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                   'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[1], None, None)',
                   "rgb_u8_to_yuv420(rs[1], 'nv12', yuv[1])"],
 'crop': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, (2, 2))',
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, (2, 2))',
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
          'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, (2, 2))',
          'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
          'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, (2, 2))',
          'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'crop_bgr': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, True, (2, 2))',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, True, (2, 2))',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
              'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, True, (2, 2))',
              'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
              'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, True, (2, 2))',
              'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'crop_nv12': ["stream_frame_in_yuv(inp[0], 'nv12', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, (2, 2))",
               'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
               "stream_frame_in_yuv(inp[1], 'nv12', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, (2, 2))",
               'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
               "stream_frame_in_yuv(inp[0], 'nv12', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, (2, 2))",
               'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
               "stream_frame_in_yuv(inp[1], 'nv12', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, (2, 2))",
               'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'out_frame': ["fill_black(pad[0], None, 'bt601')",
               "fill_black(pad[1], None, 'bt601')",
               'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
               'step_into(lr[0], lr[1], hr[1], hr[0], None)',
               'float_to_uint8_nhwc_window(hr[0], pad[0], (4, 4))',
               'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
               'step_into(lr[1], lr[0], hr[0], hr[1], None)',
               'float_to_uint8_nhwc_window(hr[1], pad[1], (4, 4))',
               'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
               'step_into(lr[0], lr[1], hr[1], hr[0], None)',
               'float_to_uint8_nhwc_window(hr[0], pad[0], (4, 4))',
               'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
               'step_into(lr[1], lr[0], hr[0], hr[1], None)',
               'float_to_uint8_nhwc_window(hr[1], pad[1], (4, 4))'],
 'out_frame_nv12': ["fill_black(yuv[0], 'nv12', 'bt601')",
                    "fill_black(yuv[1], 'nv12', 'bt601')",
                    'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                    'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                    "rgb_to_yuv('nv12', 'bt601', u8[0], None, yuv[0], (4, 4))",
                    'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                    'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                    "rgb_to_yuv('nv12', 'bt601', u8[1], None, yuv[1], (4, 4))",
                    'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                    'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                    "rgb_to_yuv('nv12', 'bt601', u8[0], None, yuv[0], (4, 4))",
                    'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                    'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                    "rgb_to_yuv('nv12', 'bt601', u8[1], None, yuv[1], (4, 4))"],
 'out_frame_p010': ["fill_black(yuv[0], 'p010', 'bt601')",
                    "fill_black(yuv[1], 'p010', 'bt601')",
                    'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                    'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                    "rgb_to_yuv('p010', 'bt601', None, hr[0], yuv[0], (4, 4))",
                    'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                    'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                    "rgb_to_yuv('p010', 'bt601', None, hr[1], yuv[1], (4, 4))",
                    'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                    'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                    "rgb_to_yuv('p010', 'bt601', None, hr[0], yuv[0], (4, 4))",
                    'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                    'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                    "rgb_to_yuv('p010', 'bt601', None, hr[1], yuv[1], (4, 4))"],
 'out_frame_size': ["fill_black(pad[0], None, 'bt601')",
                    "fill_black(pad[1], None, 'bt601')",
                    'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                    'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                    'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), pad[0], None, (8, '
                    '12))',
                    'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                    'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                    'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), pad[1], None, (8, '
                    '12))',
                    'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                    'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                    'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), pad[0], None, (8, '
                    '12))',
                    'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                    'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                    'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), pad[1], None, (8, '
                    '12))'],
 'out_frame_size_p010': ["fill_black(yuv[0], 'p010', 'bt601')",
                         "fill_black(yuv[1], 'p010', 'bt601')",
                         'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                         'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                         'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[0], '
                         'None)',
                         "rgb_to_yuv('p010', 'bt601', None, rs[0], yuv[0], (8, 12))",
                         'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                         'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                         'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[1], '
                         'None)',
                         "rgb_to_yuv('p010', 'bt601', None, rs[1], yuv[1], (8, 12))",
                         'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
                         'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                         'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[0], '
                         'None)',
                         "rgb_to_yuv('p010', 'bt601', None, rs[0], yuv[0], (8, 12))",
                         'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
                         'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                         'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), None, rs[1], '
                         'None)',
                         "rgb_to_yuv('p010', 'bt601', None, rs[1], yuv[1], (8, 12))"],
 'in_size': ["stream_frame_in_resample(inp[0], None, 'bt601', mask[0], lr[0], lr[1], hr[1], 4, (in_tables[0][0], "
             'in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
             'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
             "stream_frame_in_resample(inp[1], None, 'bt601', mask[1], lr[1], lr[0], hr[0], 4, (in_tables[0][0], "
             'in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
             'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
             "stream_frame_in_resample(inp[0], None, 'bt601', mask[0], lr[0], lr[1], hr[1], 4, (in_tables[0][0], "
             'in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
             'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
             "stream_frame_in_resample(inp[1], None, 'bt601', mask[1], lr[1], lr[0], hr[0], 4, (in_tables[0][0], "
             'in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
             'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'in_size_nv12': ["stream_frame_in_resample(inp[0], 'nv12', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
                  'scene_cut(lr[0], lr[1], mask[0], 10.0, prev_mafd, work, score[0], cut[0])',
                  'stream_frame_in(None, cut[0], lr[0], lr[1], hr[1], 4, False, None)',
                  'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                  "stream_frame_in_resample(inp[1], 'nv12', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
                  'scene_cut(lr[1], lr[0], mask[1], 10.0, prev_mafd, work, score[1], cut[1])',
                  'stream_frame_in(None, cut[1], lr[1], lr[0], hr[0], 4, False, None)',
                  'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                  "stream_frame_in_resample(inp[0], 'nv12', 'bt601', mask[0], lr[0], lr[1], hr[1], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
                  'scene_cut(lr[0], lr[1], mask[0], 10.0, prev_mafd, work, score[0], cut[0])',
                  'stream_frame_in(None, cut[0], lr[0], lr[1], hr[1], 4, False, None)',
                  'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                  "stream_frame_in_resample(inp[1], 'nv12', 'bt601', mask[1], lr[1], lr[0], hr[0], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, None)',
                  'scene_cut(lr[1], lr[0], mask[1], 10.0, prev_mafd, work, score[1], cut[1])',
                  'stream_frame_in(None, cut[1], lr[1], lr[0], hr[0], 4, False, None)',
                  'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'in_size_crop': ["stream_frame_in_resample(inp[0], None, 'bt601', mask[0], lr[0], lr[1], hr[1], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, (2, '
                  '2))',
                  'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                  "stream_frame_in_resample(inp[1], None, 'bt601', mask[1], lr[1], lr[0], hr[0], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, (2, '
                  '2))',
                  'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                  "stream_frame_in_resample(inp[0], None, 'bt601', mask[0], lr[0], lr[1], hr[1], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, (2, '
                  '2))',
                  'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                  "stream_frame_in_resample(inp[1], None, 'bt601', mask[1], lr[1], lr[0], hr[0], 4, "
                  '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), False, (2, '
                  '2))',
                  'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'scene_cut': ['stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
               'scene_cut(lr[0], lr[1], mask[0], 10.0, prev_mafd, work, score[0], cut[0])',
               'stream_frame_in(None, cut[0], lr[0], lr[1], hr[1], 4, False, None)',
               'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
               'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
               'scene_cut(lr[1], lr[0], mask[1], 10.0, prev_mafd, work, score[1], cut[1])',
               'stream_frame_in(None, cut[1], lr[1], lr[0], hr[0], 4, False, None)',
               'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
               'stream_frame_in(inp[0], mask[0], lr[0], lr[1], hr[1], 4, False, None)',
               'scene_cut(lr[0], lr[1], mask[0], 10.0, prev_mafd, work, score[0], cut[0])',
               'stream_frame_in(None, cut[0], lr[0], lr[1], hr[1], 4, False, None)',
               'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
               'stream_frame_in(inp[1], mask[1], lr[1], lr[0], hr[0], 4, False, None)',
               'scene_cut(lr[1], lr[0], mask[1], 10.0, prev_mafd, work, score[1], cut[1])',
               'stream_frame_in(None, cut[1], lr[1], lr[0], hr[0], 4, False, None)',
               'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])'],
 'scene_cut_nv12_out_size': ["stream_frame_in_yuv420(inp[0], 'nv12', mask[0], lr[0], lr[1], hr[1], 4)",
                             'scene_cut(lr[0], lr[1], mask[0], 10.0, prev_mafd, work, score[0], cut[0])',
                             'stream_frame_in(None, cut[0], lr[0], lr[1], hr[1], 4, False, None)',
                             'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                             'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[0], '
                             'None, None)',
                             "rgb_u8_to_yuv420(rs[0], 'nv12', yuv[0])",
                             "stream_frame_in_yuv420(inp[1], 'nv12', mask[1], lr[1], lr[0], hr[0], 4)",
                             'scene_cut(lr[1], lr[0], mask[1], 10.0, prev_mafd, work, score[1], cut[1])',
                             'stream_frame_in(None, cut[1], lr[1], lr[0], hr[0], 4, False, None)',
                             'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                             'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[1], '
                             'None, None)',
                             "rgb_u8_to_yuv420(rs[1], 'nv12', yuv[1])",
                             "stream_frame_in_yuv420(inp[0], 'nv12', mask[0], lr[0], lr[1], hr[1], 4)",
                             'scene_cut(lr[0], lr[1], mask[0], 10.0, prev_mafd, work, score[0], cut[0])',
                             'stream_frame_in(None, cut[0], lr[0], lr[1], hr[1], 4, False, None)',
                             'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                             'resample(hr[0], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[0], '
                             'None, None)',
                             "rgb_u8_to_yuv420(rs[0], 'nv12', yuv[0])",
                             "stream_frame_in_yuv420(inp[1], 'nv12', mask[1], lr[1], lr[0], hr[0], 4)",
                             'scene_cut(lr[1], lr[0], mask[1], 10.0, prev_mafd, work, score[1], cut[1])',
                             'stream_frame_in(None, cut[1], lr[1], lr[0], hr[0], 4, False, None)',
                             'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                             'resample(hr[1], (tables[0][0], tables[0][1]), (tables[1][0], tables[1][1]), rs[1], '
                             'None, None)',
                             "rgb_u8_to_yuv420(rs[1], 'nv12', yuv[1])"],
 'pad_reflect': ['stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                 'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                 'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                 'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                 'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                 'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                 'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                 'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                 'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                 'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                 'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                 'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                 'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                 'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                 'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                 'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                 'stream_frame_in(inp[0], None, ring[0], lr[0], hr[0], 4, False, None)',
                 'stream_frame_in(inp[1], None, ring[1], lr[0], hr[0], 4, False, None)',
                 'stream_frame_in(inp[0], None, ring[2], lr[0], hr[0], 4, False, None)'],
 'pad_replicate': ['stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                   'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                   'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                   'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                   'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                   'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                   'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                   'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                   'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                   'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                   'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                   'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                   'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                   'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                   'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                   'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                   'stream_frame_in(inp[0], None, ring[0], lr[0], hr[0], 4, False, None)',
                   'stream_frame_in(inp[1], None, ring[1], lr[0], hr[0], 4, False, None)',
                   'stream_frame_in(inp[0], None, ring[2], lr[0], hr[0], 4, False, None)'],
 'pad_reflect_cut': ['stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                     'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                     'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                     'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                     'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                     'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                     'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                     'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                     'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                     'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                     'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                     'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                     'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                     'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                     'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                     'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                     'stream_frame_in(inp[0], None, ring[0], lr[0], hr[0], 4, False, None)',
                     'scene_cut(ring[0], ring[3], in_mask, 10.0, prev_mafd, work, rep_ring[0], rep_ring[0]+16)',
                     'stream_frame_in(inp[1], None, ring[1], lr[0], hr[0], 4, False, None)',
                     'scene_cut(ring[1], ring[0], None, 10.0, prev_mafd, work, rep_ring[1], rep_ring[1]+16)',
                     'stream_frame_in(inp[0], None, ring[2], lr[0], hr[0], 4, False, None)',
                     'scene_cut(ring[2], ring[1], None, 10.0, prev_mafd, work, rep_ring[2], rep_ring[2]+16)'],
 'pad_replicate_cut': ['stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                       'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                       'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                       'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                       'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                       'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                       'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                       'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                       'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                       'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                       'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                       'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                       'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                       'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                       'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                       'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                       'stream_frame_in(inp[0], None, ring[0], lr[0], hr[0], 4, False, None)',
                       'scene_cut(ring[0], ring[3], in_mask, 10.0, prev_mafd, work, rep_ring[0], rep_ring[0]+16)',
                       'stream_frame_in(inp[1], None, ring[1], lr[0], hr[0], 4, False, None)',
                       'scene_cut(ring[1], ring[0], None, 10.0, prev_mafd, work, rep_ring[1], rep_ring[1]+16)',
                       'stream_frame_in(inp[0], None, ring[2], lr[0], hr[0], 4, False, None)',
                       'scene_cut(ring[2], ring[1], None, 10.0, prev_mafd, work, rep_ring[2], rep_ring[2]+16)'],
 'pad_f32_cut': ['stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                 'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                 'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                 'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                 'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                 'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                 'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                 'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                 'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                 'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                 'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                 'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                 'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                 'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                 'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                 'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                 'scene_cut(ring[0], ring[3], in_mask, 10.0, prev_mafd, work, rep_ring[0], rep_ring[0]+16)',
                 'scene_cut(ring[1], ring[0], None, 10.0, prev_mafd, work, rep_ring[1], rep_ring[1]+16)',
                 'scene_cut(ring[2], ring[1], None, 10.0, prev_mafd, work, rep_ring[2], rep_ring[2]+16)'],
 'pad_nv12_crop_p010': ['stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                        'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                        "rgb_to_yuv('p010', 'bt601', None, hr[0], yuv[0], None)",
                        'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                        'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                        "rgb_to_yuv('p010', 'bt601', None, hr[1], yuv[1], None)",
                        'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                        'step_into(lr[0], lr[1], hr[1], hr[0], u8[0])',
                        "rgb_to_yuv('p010', 'bt601', None, hr[0], yuv[0], None)",
                        'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                        'step_into(lr[1], lr[0], hr[0], hr[1], u8[1])',
                        "rgb_to_yuv('p010', 'bt601', None, hr[1], yuv[1], None)",
                        'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                        'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                        'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                        'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                        'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                        'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                        'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                        'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                        "stream_frame_in_yuv(inp[0], 'nv12', 'bt601', None, ring[0], lr[0], hr[0], 4, (2, 2))",
                        "stream_frame_in_yuv(inp[1], 'nv12', 'bt601', None, ring[1], lr[0], hr[0], 4, (2, 2))",
                        "stream_frame_in_yuv(inp[0], 'nv12', 'bt601', None, ring[2], lr[0], hr[0], 4, (2, 2))"],
 'pad_in_size_out_frame': ["fill_black(pad[0], None, 'bt601')",
                           "fill_black(pad[1], None, 'bt601')",
                           'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                           'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                           'float_to_uint8_nhwc_window(hr[0], pad[0], (4, 4))',
                           'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                           'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                           'float_to_uint8_nhwc_window(hr[1], pad[1], (4, 4))',
                           'stream_gather(ring, mtab[0], whr[0], lr[0], lr[1], hr[1], 4)',
                           'step_into(lr[0], lr[1], hr[1], hr[0], None)',
                           'float_to_uint8_nhwc_window(hr[0], pad[0], (4, 4))',
                           'stream_gather(ring, mtab[1], whr[0], lr[1], lr[0], hr[0], 4)',
                           'step_into(lr[1], lr[0], hr[0], hr[1], None)',
                           'float_to_uint8_nhwc_window(hr[1], pad[1], (4, 4))',
                           'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                           'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                           'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                           'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                           'stream_gather(ring, wtab[0], None, wlr[0], wlr[1], whr[1], 4)',
                           'step_into(wlr[0], wlr[1], whr[1], whr[0], None)',
                           'stream_gather(ring, wtab[1], None, wlr[1], wlr[0], whr[0], 4)',
                           'step_into(wlr[1], wlr[0], whr[0], whr[1], None)',
                           "stream_frame_in_resample(inp[0], None, 'bt601', None, ring[0], lr[0], hr[0], 4, "
                           '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), '
                           'False, None)',
                           "stream_frame_in_resample(inp[1], None, 'bt601', None, ring[1], lr[0], hr[0], 4, "
                           '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), '
                           'False, None)',
                           "stream_frame_in_resample(inp[0], None, 'bt601', None, ring[2], lr[0], hr[0], 4, "
                           '(in_tables[0][0], in_tables[0][1]), (in_tables[1][0], in_tables[1][1]), (32, 48), '
                           'False, None)']}


@pytest.fixture(scope='module')
def net():
    torch.manual_seed(0)
    return T.FRNet(3, 3, 64, 1, 'BD', 4).to(DEV).eval()


@pytest.mark.parametrize('case', [c for c, _ in CASES])
def test_stream_launch_plan(net, monkeypatch, case):
    kw = dict(CASES)[case]
    assert launch_plan(net, monkeypatch, **kw) == EXPECTED[case]
