"""rqvae -- drop-in, H100-native replacement for the sampling hot path of kakaobrain/rq-vae-transformer.

Same import paths and class surface as the reference's ``rqvae`` package for the path in SURVEY.md section 8
(``rqvae.models.create_model``, ``RQVAE``, ``RQBottleneck``, ``RQTransformer``, ``rqvae.utils.utils``), but every
numeric op runs in hand-written sm_90a CUDA kernels behind the C ABI of ``include/rqb200.h``
(``csrc/librqb200.so``).  There is no CPU / eager fallback: calling a compute method without the native library
or on non-CUDA tensors raises.
"""
__version__ = "0.1.0"
