"""open_muse_b200 -- the H100 (sm_90a) hot path of huggingface/open-muse behind the reference's Python surface.

    from open_muse_b200 import MaskGitTransformer, MaskGitVQGAN

See DESIGN.md (scope, kernels, parity) and INTEGRATION.md (how the reference binds it).
"""
__version__ = "0.1.0"

from .modeling_ema import EMAModel  # noqa: F401
from .modeling_maskgit_vqgan import MaskGitVQGAN  # noqa: F401
from .modeling_taming_vqgan import VQGANModel  # noqa: F401
from .modeling_transformer import MaskGitTransformer  # noqa: F401
from .modeling_transformer_v2 import MaskGiTUViT_v2  # noqa: F401

MaskGiTUViT = MaskGiTUViT_v2  # the reference's alias (muse/modeling_transformer.py:41)
from .pipeline_muse import PipelineMuse, PipelineMuseInpainting  # noqa: F401
from .sampling import get_mask_chedule  # noqa: F401

from .optim import FusedAdamW  # noqa: F401,E402
