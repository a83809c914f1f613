"""salience-detr_b200: H100-native (sm_90a) Salience-DETR encoder hot path.

Hierarchical salience top-k token filter + multi-scale deformable self-attention over the selected
tokens, behind the reference's own module / operator boundary (xiuqhou/Salience-DETR,
models/bricks/{salience_transformer,ms_deform_attn}.py).  Python/PyTorch host code calling hand-written
CUDA through the C-ABI in ``include/sdetr_b200.h``; no Triton, no CPU or PyTorch fallback.

The directory name contains a hyphen; ``import salience_detr_b200`` works through the loader shim
``salience_detr_b200.py`` at the repository root.
"""
from . import cabi  # noqa: F401
from .build import build as build_library  # noqa: F401
from .ms_deform_attn import (  # noqa: F401
    _C,
    MultiScaleDeformableAttention,
    MultiScaleDeformableAttnFunction,
    ms_deform_attn_backward,
    ms_deform_attn_forward,
)
from . import gemm  # noqa: F401
from .position_encoding import PositionEmbeddingSine  # noqa: F401
from .criterion import SalienceCriterion, load_reference_checkpoint, sigmoid_focal_loss  # noqa: F401
from .set_criterion import HungarianMatcher, HybridSetCriterion  # noqa: F401
from .denoising import GenerateCDNQueries, compute_dn_loss  # noqa: F401
from .postprocess import PostProcess  # noqa: F401
from .decoder import (  # noqa: F401
    MLP,
    SalienceTransformerDecoder,
    SalienceTransformerDecoderLayer,
    get_sine_pos_embed,
    inverse_sigmoid,
)
from .neck import (  # noqa: F401
    Conv2dNormActivation,
    CSPRepPluXLayer,
    RepVGGPluXNetwork,
    RepVggPluXBlock,
    SqueezeAndExcitation,
)
from .channel_mapper import ChannelMapper, level_views, tokens_of  # noqa: F401
from .salience_transformer import (  # noqa: F401
    EncoderPlan,
    MaskPredictor,
    PositionEmbeddingLearned,
    SalienceTransformer,
    SalienceTransformerEncoder,
    SalienceTransformerEncoderLayer,
    flatten_levels,
)

__version__ = "0.1.0"
