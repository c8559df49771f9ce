"""Drop-in ``muse`` package: put ``open_muse_b200/compat`` on PYTHONPATH and the reference's
``from muse import MaskGitTransformer, MaskGitVQGAN, PipelineMuse`` / ``from muse.sampling import cosine_schedule``
(training/train_maskgit_imagenet.py:30-33) resolve to the H100 implementations."""
__version__ = "0.0.1"

from open_muse_b200 import (  # noqa: F401
    EMAModel,
    MOVQ,
    MaskGiTUViT,
    MaskGitTransformer,
    MaskGiTUViT_v2,
    MaskGitVQGAN,
    PipelineMuse,
    PipelineMuseInpainting,
    VQGANModel,
    get_mask_chedule,
)
from open_muse_b200 import modeling_transformer_v2, sampling  # noqa: F401
from . import logging, lr_schedulers  # noqa: F401,E402
from open_muse_b200.modeling_paella_vq import PaellaVQModel  # noqa: F401,E402
