"""RQVAE at any image size, host side (no GPU): encode / decode / forward / get_codes / get_soft_codes refuse an input that is not 4-D,
has the wrong channel count, or an extent that is not a positive multiple of the downsampling factor f = 2^(len(ch_mult) - 1), with
ValueError before any native call; the latent / image shape arithmetic; and the tensor-core attention diagnostic's refusals."""
import ctypes

import pytest
import torch

from oracle.zoo import VAE_ZOO, vae_ddconfig
from rqvae import _native as N
from rqvae.models import create_model
from tests.helpers import vae_config


def cpu_vae(name):
    with torch.device("meta"):
        model, _ = create_model(vae_config(name))
    return model.to_empty(device="cpu").eval()


@pytest.mark.parametrize("name,f", [("tiny", 4), ("tiny_attn_mid", 8), ("imagenet", 32)])
def test_downsample_factor(name, f):
    model = cpu_vae(name)
    assert model.downsample_factor() == f == 2 ** (len(vae_ddconfig(**VAE_ZOO[name])["ch_mult"]) - 1)
    assert model.ddconfig["resolution"] // f == model.code_shape[0]


def test_shape_arithmetic():
    """the extents the checks accept are exactly the positive multiples of f, and the latent of an accepted image is its extent / f"""
    model = cpu_vae("tiny")
    f = model.downsample_factor()
    for H in range(0, 41):
        for W in (4, 12, 20):
            x = torch.zeros(1, 3, H, W)
            if H >= 1 and H % f == 0:
                assert model._check_input(x, 3, "image", f) == (H, W)
                assert (H // f, W // f) == (H // 4, W // 4)
            else:
                with pytest.raises(ValueError):
                    model._check_input(x, 3, "image", f)


BAD_IMAGES = {
    "3-D": (3, 16, 16),
    "5-D": (1, 1, 3, 16, 16),
    "channels": (2, 4, 16, 16),
    "height not a multiple of f": (2, 3, 18, 16),
    "width not a multiple of f": (2, 3, 16, 6),
    "empty extent": (2, 3, 0, 16),
    "empty batch": (0, 3, 16, 16),
}


@pytest.mark.parametrize("why", sorted(BAD_IMAGES))
@pytest.mark.parametrize("method", ["encode", "forward", "get_codes", "get_soft_codes"])
def test_image_input_refused_before_native_call(why, method):
    model = cpu_vae("tiny")
    with pytest.raises(ValueError):
        getattr(model, method)(torch.zeros(BAD_IMAGES[why]))


BAD_LATENTS = {
    "3-D": (2, 16, 256),
    "embed_dim": (2, 4, 4, 128),
    "NCHW instead of NHWC": (2, 256, 4, 4),
    "empty extent": (2, 0, 4, 256),
}


@pytest.mark.parametrize("why", sorted(BAD_LATENTS))
def test_latent_input_refused_before_native_call(why):
    model = cpu_vae("tiny")
    with pytest.raises(ValueError):
        model.decode(torch.zeros(BAD_LATENTS[why]))


@pytest.mark.parametrize("shape", [(1, 3, 8, 8), (2, 3, 12, 20), (1, 3, 16, 16)])
def test_valid_image_reaches_the_cuda_check(shape):
    """an acceptable image passes the shape checks and is refused only for being on the CPU (NativeError, not ValueError)"""
    model = cpu_vae("tiny")
    with pytest.raises(N.NativeError):
        model.encode(torch.zeros(shape))


@pytest.mark.parametrize("shape", [(1, 1, 1, 256), (2, 3, 5, 256)])
def test_valid_latent_reaches_the_cuda_check(shape):
    model = cpu_vae("tiny")
    with pytest.raises(N.NativeError):
        model.decode(torch.zeros(shape))


def test_decode_code_keeps_the_configured_code_shape():
    model = cpu_vae("tiny")
    with pytest.raises(AssertionError):
        model.decode_code(torch.zeros(1, 3, 5, 4, dtype=torch.int64))


@pytest.mark.parametrize("B,HW,C", [(1, 2048, 96), (1, 2048, 640), (1, 2048, 64), (0, 2048, 512), (1, 0, 512)])
def test_attention_tc_diagnostic_refusals(B, HW, C):
    """head dimensions other than 128 | 256 | 384 | 512, and empty shapes, are refused before any CUDA call"""
    buf = ctypes.create_string_buffer(64)            # stands in for the device pointers; never dereferenced
    assert N.lib().rqb200_dbg_vae_attn_tc(buf, buf, B, HW, C, None) == N.EINVAL
