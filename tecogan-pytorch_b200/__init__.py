"""tecogan-pytorch_b200: the FRNet generator hot path of TecoGAN-PyTorch on hand-written sm_90a
kernels, behind the reference's Python surface.  Import with
``importlib.import_module('tecogan-pytorch_b200')`` or through the ``tecogan_b200`` alias module
at the repo root."""
from .lib import TecoganB200Error, load as load_library, LIB_PATH  # noqa: F401
from .networks import FRNet, FNet, SRNet, ResidualBlock, BaseSequenceGenerator  # noqa: F401
from .net_utils import (space_to_depth, backward_warp, get_upsampling_func,  # noqa: F401
                        BicubicUpsampler, BilinearUpsampler)
from .data_utils import create_kernel, downsample_bd  # noqa: F401
from .factory import define_generator  # noqa: F401
from . import engine  # noqa: F401
from .engine import infer_clips, ClipEngine, release_engines, StreamEngine, VideoStream  # noqa: F401
from .sharding import clips_for_rank  # noqa: F401
from .autograd import st_discriminator_input  # noqa: F401
from . import reducer  # noqa: F401
from . import metrics  # noqa: F401
from .reducer import FlatGradientReducer  # noqa: F401

__all__ = ['FRNet', 'FNet', 'SRNet', 'define_generator', 'space_to_depth', 'backward_warp',
           'get_upsampling_func', 'BicubicUpsampler', 'infer_clips', 'ClipEngine', 'VideoStream',
           'clips_for_rank', 'st_discriminator_input', 'FlatGradientReducer', 'load_library', 'TecoganB200Error', 'create_kernel', 'downsample_bd',
           'metrics']
