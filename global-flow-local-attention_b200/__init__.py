"""gfla_b200 -- H100-native (sm_90a) warping hot path of Global-Flow-Local-Attention.

The package keeps its historical name ``gfla_b200``.

The directory is called ``global-flow-local-attention_b200`` (not an importable
name), so the repo root carries ``gfla_b200.py`` which loads it under the module
name ``gfla_b200``.  Public surface = the reference's own classes:

    BlockExtractor / BlockExtractorFunction        (block_extractor.py)
    LocalAttnReshape / LocalAttnReshapeFunction    (local_attn_reshape.py)
    Resample2d / Resample2dFunction                (resample2d.py)
    ExtractorAttn                                  (base_function.py:790-818)
    AffineRegularizationLoss / MultiAffineRegularizationLoss   (external_function.py:12-77)
    PerceptualCorrectness                          (external_function.py:222-284, on the fused Resample2dCosine op)
plus the fused ops ``local_attention`` / ``LocalAttnFunction`` and ``patch_conv`` / ``PatchConvFunction``
(ExtractorAttn's source-half conv without the block tensor), and ``compat.install()`` for the legacy
extension-module names.
"""
from .block_extractor import BlockExtractor, BlockExtractorFunction
from .extractor_attn import ExtractorAttn, LocalAttnFunction, PatchConvFunction, local_attention, patch_conv
from .local_attn_reshape import LocalAttnReshape, LocalAttnReshapeFunction
from .losses import AffineRegularizationLoss, MultiAffineRegularizationLoss, PerceptualCorrectness
from .resample2d import Resample2d, Resample2dCosine, Resample2dCosineFunction, Resample2dFunction
from . import compat, functional, losses, sharding  # noqa: F401

__all__ = ["BlockExtractor", "BlockExtractorFunction", "LocalAttnReshape", "LocalAttnReshapeFunction", "Resample2d",
           "Resample2dFunction", "ExtractorAttn", "LocalAttnFunction", "local_attention", "PatchConvFunction", "patch_conv",
           "AffineRegularizationLoss",
           "MultiAffineRegularizationLoss", "PerceptualCorrectness", "Resample2dCosine", "Resample2dCosineFunction", "compat", "functional",
           "sharding"]
