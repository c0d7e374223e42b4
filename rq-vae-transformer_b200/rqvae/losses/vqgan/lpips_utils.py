"""Where the LPIPS weight files are found (reference: rqvae/losses/vqgan/lpips_utils.py).  Nothing is ever downloaded: a file that is
not in one of the places looked at raises FileNotFoundError naming every path and the reference's URL."""
import hashlib
import os

import torch

URL_MAP = {
    "vgg_lpips": "https://heibox.uni-heidelberg.de/f/607503859c864bc1b30b/?dl=1"
}

CKPT_MAP = {
    "vgg_lpips": "vgg.pth"
}

MD5_MAP = {
    "vgg_lpips": "d507d7349b931f0638a25a48a722f98a"
}

# torchvision's ImageNet VGG16, where models.vgg16(pretrained=True) caches it
VGG16_URL = "https://download.pytorch.org/models/vgg16-397923af.pth"


def md5_hash(path):
    with open(path, "rb") as f:
        content = f.read()
    return hashlib.md5(content).hexdigest()


def ckpt_candidates(name, root=None):
    """the paths get_ckpt_path looks at, in order: <root>/<file> when root is given; else the reference's
    <package>/rqvae/losses/vqgan/.caches/<file>, then <torch.hub.get_dir()>/checkpoints/<file>"""
    f = CKPT_MAP[name]
    if root is not None:
        return [os.path.join(root, f)]
    return [os.path.join(os.path.dirname(os.path.abspath(__file__)), ".caches", f),
            os.path.join(torch.hub.get_dir(), "checkpoints", f)]


def get_ckpt_path(name, root=None, check=False):
    """the first existing file of ckpt_candidates(name, root); with check, its md5 must be the reference's (ValueError otherwise)"""
    if name not in URL_MAP:
        raise ValueError("get_ckpt_path: unknown checkpoint %r (known: %s)" % (name, ", ".join(URL_MAP)))
    paths = ckpt_candidates(name, root)
    for path in paths:
        if os.path.isfile(path):
            if check and md5_hash(path) != MD5_MAP[name]:
                raise ValueError("get_ckpt_path: %s has md5 %s, expected %s" % (path, md5_hash(path), MD5_MAP[name]))
            return path
    raise FileNotFoundError("rqb200: the %s weights are not at %s.  This package never downloads; copy %s (from %s) to one of those "
                            "paths" % (name, " or ".join(paths), CKPT_MAP[name], URL_MAP[name]))


def vgg16_weights_path():
    """where torchvision's models.vgg16(pretrained=True) caches the ImageNet VGG16: <torch.hub.get_dir()>/checkpoints/<file>
    (TORCH_HOME relocates it)"""
    return os.path.join(torch.hub.get_dir(), "checkpoints", os.path.basename(VGG16_URL))
