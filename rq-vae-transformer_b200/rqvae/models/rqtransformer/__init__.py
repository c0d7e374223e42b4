"""Stage-2 prior: parameter tree + native AR engine binding (see transformers.py)."""
from .configs import RQTransformerConfig  # noqa: F401  (re-exported for callers that build structured configs)
from .transformers import RQTransformer  # noqa: F401
from .rejection import rejection_sample  # noqa: F401


def get_rqtransformer(config):
    """factory used by rqvae.models.create_model for ``type: rq-transformer`` (same role as the reference's getter)"""
    model = RQTransformer(config)
    return model
