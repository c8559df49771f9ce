"""Drop-in ``muse`` package: put ``open_muse_b200/compat`` on PYTHONPATH and the reference's
``from muse import MaskGitTransformer, MaskGitVQGAN, PipelineMuse`` / ``from muse.sampling import cosine_schedule``
(training/train_maskgit_imagenet.py:30-33) resolve to the H100 implementations."""
__version__ = "0.0.1"

from open_muse_b200 import (  # noqa: F401
    EMAModel,
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


class _OutOfScopeTokenizer:
    """MOVQ / PaellaVQModel are other tokenizers the training scripts import by name (training/train_muse.py:49-58,
    train_maskgit_imagenet.py:38); they are outside this package's hot path (DESIGN.md section 7) and fail loudly if a
    config actually selects them."""

    def __init__(self, *a, **k):
        raise NotImplementedError(f"open_muse_b200: {type(self).__name__} is not part of the H100 hot path; use "
                                  "MaskGitVQGAN (model.vq_model.type: maskgit_vqgan) or VQGANModel (taming)")

    @classmethod
    def from_pretrained(cls, *a, **k):
        return cls()


class MOVQ(_OutOfScopeTokenizer):
    pass


class PaellaVQModel(_OutOfScopeTokenizer):
    pass
