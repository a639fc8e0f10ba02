"""Drop-in for `from diffuser_engine.models.modeling_vae import CVVAEModel`
(reference pipelines/pipeline_stable_diffusion.py:41), backed by the sm_90a engine."""
from cvvae_b200.modeling_vae import (AutoencoderKLOutput, CVVAEModel, CVVAESD3Model, DecoderOutput,  # noqa: F401
                                     DiagonalGaussianDistribution)

__all__ = ["CVVAEModel", "CVVAESD3Model", "DiagonalGaussianDistribution", "DecoderOutput", "AutoencoderKLOutput"]
