"""iaf_b200: the IAF posterior's masked-autoregressive step (openai/iaf down_iaf2_nl /
up_iaf2_nl) as hand-written sm_90a (H100) CUDA behind the reference's python signatures."""
from .ops import IAFOperator, ar_multiconv2d, iaf_step, multiconv2d  # noqa: F401

__all__ = ["IAFOperator", "ar_multiconv2d", "multiconv2d", "iaf_step"]
