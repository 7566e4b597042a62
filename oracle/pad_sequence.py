"""Temporal padding of a test sequence: BaseModel.pad_sequence (base_model.py:230-251) restated with its two options
(test.yml's num_pad_front and padding_mode) as arguments, and `reference_pad_sequence`, the unmodified reference
method where oracle/_ref holds the reference install.

FRNet.stream(pad_front=p, padding_mode=...) makes, for every shot, the frames of
infer_sequence(pad_sequence(shot, q, padding_mode)[0])[q:].  `gather` states the contract of tg_stream_gather, the
launch that assembles each of its steps' inputs from the ring of decoded frames.
"""
import types

import torch


def pad_sequence(lr_data, num_pad_front, padding_mode='reflect'):
    """lr_data tchw -> (padded tchw, num_pad_front): 'reflect' prepends lr_data[1:1+p] reversed, 'replicate' p copies
    of lr_data[0].  Like the reference, p < t is asserted."""
    assert num_pad_front < lr_data.size(0)
    if padding_mode == 'reflect':
        lr_data = torch.cat([lr_data[1:1 + num_pad_front, ...].flip(0), lr_data], dim=0)
    elif padding_mode == 'replicate':
        lr_data = torch.cat([lr_data[:1, ...].expand(num_pad_front, -1, -1, -1), lr_data], dim=0)
    else:
        raise ValueError(f'Unrecognized padding mode: {padding_mode}')
    return lr_data, num_pad_front


def reference_pad_sequence():
    """The reference's own BaseModel.pad_sequence as a function of (lr_data, num_pad_front, padding_mode), or None
    where the reference is not installed."""
    import refimport
    if not refimport.available():
        return None
    refimport.import_models()
    from models.base_model import BaseModel

    def pad(lr_data, num_pad_front, padding_mode='reflect'):
        holder = types.SimpleNamespace(opt={'test': {'padding_mode': padding_mode, 'num_pad_front': num_pad_front}})
        return BaseModel.pad_sequence(holder, lr_data)
    return pad


KEEP, ZERO, LOAD = 0, 1, 2               # TG_GATHER_KEEP / _ZERO / _LOAD


def gather(ring, table, warm_hr, lr_curr, lr_prev, hr_prev):
    """tg_stream_gather's contract on NumPy arrays, in place: ring [depth,n,c,h,w], table int [3n] (cur, mode, prev
    per slot), warm_hr [n,c,H,W] or None, lr_curr / lr_prev [n,c,h,w], hr_prev [n,c,H,W]."""
    depth, n = ring.shape[:2]
    cur, mode, prev = table[:n], table[n:2 * n], table[2 * n:]
    for k in range(n):
        if 0 <= cur[k] < depth:
            lr_curr[k] = ring[cur[k], k]
        if mode[k] == ZERO:
            lr_prev[k] = 0
            hr_prev[k] = 0
        elif mode[k] == LOAD and warm_hr is not None:
            lr_prev[k] = ring[prev[k], k] if 0 <= prev[k] < depth else 0
            hr_prev[k] = warm_hr[k]
