"""maskdit_b200 — H100-native (sm_90a) implementation of the MaskDiT training / sampling hot path.

Public surface mirrors the reference registries (models/maskdit.py:709-715,779-781, train_utils/loss.py:66-68,
sample.py:30-66): `Precond_models`, `DiT_models`, `Losses`, `edm_sampler`.
"""
__version__ = "0.1.0"
