"""VGG19 perceptual-loss features on the library's kernels: a drop-in for the reference's VGGFeatureExtractor
(codes/models/networks/vgg_nets.py), used by VSRGANModel's feature loss (vsrgan_model.py:225-238).

Every conv of vgg19.features runs on tg_conv_tcgen05 with its ReLU in the epilogue (NHWC fp16, 64 ... 512 channels),
every max-pool on tg_maxpool2x2_nhwc_f16, and the input normalisation (x - mean) / std on tg_grad_pack_ex_nhwc_f16.
The requested features come back as NCHW fp32 tensors.  Under autograd the whole extractor is one
torch.autograd.Function (autograd.VGGFeaturesFunction) whose backward produces the input gradient only: VGG's
parameters are frozen, and their gradients are never formed.  DESIGN.md section 10 describes the layout, the taps and
the loss scaling.
"""
import torch
import torch.nn as nn

from . import lib as L
from . import ops

MIN_SIDE = 16     # four floor max-pools must leave relu5_4 at least 1 x 1


def _plan(features):
    """vgg19.features -> ([(conv index, relu index, pool follows)], {relu index: unit}) ; anything but the
    Conv2d(3x3, pad 1) + ReLU (+ MaxPool2d(2, 2)) pattern of torchvision's VGG19 is rejected"""
    mods = list(features)
    units, relu_unit = [], {}
    i = 0
    while i < len(mods):
        conv = mods[i]
        if not (isinstance(conv, nn.Conv2d) and conv.kernel_size == (3, 3) and conv.padding == (1, 1)
                and conv.stride == (1, 1) and conv.bias is not None and i + 1 < len(mods)
                and isinstance(mods[i + 1], nn.ReLU)):
            raise ValueError(f'VGGFeatureExtractor: features[{i}] is {conv!r}, expected a 3x3 conv followed by a ReLU')
        pool = i + 2 < len(mods) and isinstance(mods[i + 2], nn.MaxPool2d)
        if pool and not (mods[i + 2].kernel_size in (2, (2, 2)) and mods[i + 2].stride in (2, (2, 2))
                         and not mods[i + 2].ceil_mode and mods[i + 2].padding in (0, (0, 0))):
            raise ValueError(f'VGGFeatureExtractor: features[{i + 2}] is {mods[i + 2]!r}, expected MaxPool2d(2, 2)')
        relu_unit[i + 1] = len(units)
        units.append((i, i + 1, pool))
        i += 3 if pool else 2
    return units, relu_unit


class VGGFeatureExtractor(nn.Module):
    """The reference's VGGFeatureExtractor on the library: same constructor, parameters, buffers and state_dict keys
    (features.{i}.weight / bias, mean, std); forward(x) takes NCHW fp32 [N,3,H,W] in [0, 1] on a CUDA device and
    returns the features after the ReLUs at `feature_indexs` (sorted), NCHW fp32.  Layers beyond the deepest
    requested index are not computed."""

    def __init__(self, feature_indexs=(8, 17, 26, 35)):
        super().__init__()
        import torchvision
        self.features = torchvision.models.vgg19(pretrained=True).features
        for param in self.features.parameters():
            param.requires_grad = False
        self.feature_indexs = sorted(feature_indexs)
        self._units, relu_unit = _plan(self.features)
        for i in self.feature_indexs:
            if not isinstance(i, int) or i not in relu_unit:
                raise ValueError(f'VGGFeatureExtractor: feature index {i!r} is not a ReLU of vgg19.features '
                                 f'(ReLUs: {sorted(relu_unit)})')
        self._taps = [relu_unit[i] for i in self.feature_indexs]    # unit of each requested feature
        self._depth = max(self._taps) + 1 if self._taps else 0      # units computed
        mean = torch.FloatTensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)  # RGB
        std = torch.FloatTensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
        self.register_buffer('mean', mean)
        self.register_buffer('std', std)
        self._packed = None

    def feature_shapes(self, n, h, w):
        """[(N, C, h, w)] of the returned features for an N x 3 x h x w input (floor pools)"""
        shapes, by_unit = [], {}
        for u, (ci, _, pool) in enumerate(self._units[:self._depth]):
            by_unit[u] = (n, self.features[ci].out_channels, h, w)
            if pool:
                h, w = h // 2, w // 2
        return [by_unit[u] for u in self._taps]

    # ------------------------------------------------------------------ packed layers
    def packed_layers(self):
        """[(PackedConv, PackedDgrad)] of the computed units, repacked when the parameters changed (load_state_dict)"""
        dev = self.mean.device
        if dev.type != 'cuda':
            raise L.TecoganB200Error('VGGFeatureExtractor: the module must be on a CUDA device (no CPU fallback exists)')
        if self._packed is None or self._packed[0] != dev:
            layers = []
            for ci, _, _ in self._units[:self._depth]:
                conv = self.features[ci]
                fwd = ops.PackedConv(conv.weight, conv.bias, L.CONV_3X3, L.ACT_RELU, L.EPI_NHWC_F16)
                layers.append((fwd, ops.PackedDgrad(fwd, conv.weight)))
            self._packed = (dev, layers)
        else:
            for (ci, _, _), (fwd, dg) in zip(self._units, self._packed[1]):
                conv = self.features[ci]
                fwd.refresh(conv.weight, conv.bias)
                dg.refresh(conv.weight)
        return self._packed[1]

    def _check_input(self, x):
        if not isinstance(x, torch.Tensor) or not x.is_cuda:
            raise L.TecoganB200Error('VGGFeatureExtractor: expected a CUDA tensor (no CPU fallback exists)')
        if x.dtype != torch.float32:
            raise L.TecoganB200Error(f'VGGFeatureExtractor: expected float32 input, got {x.dtype}')
        if x.dim() != 4 or x.shape[1] != 3:
            raise L.TecoganB200Error(f'VGGFeatureExtractor: expected [N,3,H,W], got {tuple(x.shape)}')
        if x.shape[2] < MIN_SIDE or x.shape[3] < MIN_SIDE:
            raise L.TecoganB200Error(f'VGGFeatureExtractor: H and W must be at least {MIN_SIDE}, got '
                                     f'{tuple(x.shape[2:])}')
        if x.device != self.mean.device:
            raise L.TecoganB200Error(f'VGGFeatureExtractor: input on {x.device}, module on {self.mean.device}')

    def forward(self, x):
        self._check_input(x)
        from .autograd import VGGFeaturesFunction, vgg_forward
        if torch.is_grad_enabled() and x.requires_grad:
            return list(VGGFeaturesFunction.apply(self, x))
        feats, _ = vgg_forward(self, x.detach().contiguous(), keep=False)
        return feats
