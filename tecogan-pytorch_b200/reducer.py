"""Data-parallel gradient exchange of the generator (SURVEY.md 8-e / 8-f4).

The reference trains through DistributedDataParallel (base_model.py:133-139): bucketed all-reduces fired
from autograd hooks, then -- every iteration -- `reduce_log` builds a tensor from per-key `.item()` floats,
`dist.reduce`s it and `.item()`s every key again (base_model.py:156-171), and the adaptive discriminator
policy adds two scalar all-reduces + a barrier + an `.item()` (vsrgan_model.py:161-176).  Each of those is a
host round trip on the critical path of an 8-GPU step.

FlatGradientReducer is the GPU-native replacement for that exchange step: every gradient of the module
lives in ONE flat fp32 buffer (the backward kernels accumulate straight into views of it), and ONE
asynchronous NCCL all-reduce over NVLink per iteration carries the gradients AND the iteration's scalars
(losses, discriminator statistics) in its tail -- one collective, one device->host copy when the log is read.
The per-frame recurrence never leaves its GPU; this is the only exchange the path has.
"""
import torch
import torch.distributed as dist


class FlatGradientReducer:
    def __init__(self, module, n_scalars=32, process_group=None):
        self.params = [p for p in module.parameters() if p.requires_grad]
        if not self.params:
            raise ValueError('FlatGradientReducer: module has no trainable parameters')
        dev, total = self.params[0].device, sum(p.numel() for p in self.params)
        self.n_grad, self.n_scalars, self.group = total, n_scalars, process_group
        self.flat = torch.zeros(total + n_scalars, dtype=torch.float32, device=dev)
        self._views, o = [], 0
        for p in self.params:
            self._views.append(self.flat[o:o + p.numel()].view_as(p))
            o += p.numel()
        self._keys, self._work = [], None
        self.attach()

    # ------------------------------------------------------------------ gradient storage
    def attach(self):
        """(Re)point every .grad at its slice of the flat buffer; autograd then accumulates in place.
        Call after anything that replaces .grad (e.g. optimizer.zero_grad(set_to_none=True))."""
        for p, v in zip(self.params, self._views):
            p.grad = v

    def zero_grad(self):
        """one memset for all gradients and scalars (replaces optimizer.zero_grad())"""
        self.flat.zero_()
        self.attach()

    @property
    def world_size(self):
        return dist.get_world_size(self.group) if dist.is_available() and dist.is_initialized() else 1

    # ------------------------------------------------------------------ the exchange
    def all_reduce_async(self, scalars=None):
        """Start the iteration's single collective.  `scalars`: dict name -> 0-dim tensor (or float); the
        tensors are NOT synchronised with the host here."""
        scalars = scalars or {}
        if len(scalars) > self.n_scalars:
            raise ValueError(f'FlatGradientReducer: {len(scalars)} scalars > {self.n_scalars} slots')
        self._keys = list(scalars)
        tail = self.flat[self.n_grad:]
        for i, k in enumerate(self._keys):
            v = scalars[k]
            tail[i] = v.detach() if isinstance(v, torch.Tensor) else float(v)   # device-side copy, no sync
        self._work = None
        if self.world_size > 1:
            self._work = dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=self.group, async_op=True)
        return self

    def wait(self, read_scalars=True):
        """Finish the exchange: gradients (and scalars) become the mean over ranks.  Returns the averaged
        scalars as floats -- ONE device->host copy for all of them -- or None when read_scalars is False."""
        ws = self.world_size
        if self._work is not None:
            self._work.wait()
            self._work = None
            self.flat.div_(ws)
        if not read_scalars or not self._keys:
            return {} if read_scalars else None
        vals = self.flat[self.n_grad:self.n_grad + len(self._keys)].tolist()
        return dict(zip(self._keys, vals))
