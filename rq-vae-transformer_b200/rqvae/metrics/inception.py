"""InceptionV3 -- host-side mirror of rqvae/metrics/inception.py (the pytorch-fid Inception-v3) over the native Inception engine.

Boundary kept: ``InceptionV3(output_blocks, resize_input, normalize_input, requires_grad, use_fid_inception)``, its
``BLOCK_INDEX_BY_DIM`` / ``DEFAULT_BLOCK_INDEX``, ``forward(inp, return_logits=False)`` and its state_dict key layout
(``blocks.0.0.conv.weight`` ... ``fc.bias``); ``fid_inception_v3`` loads the pytorch-fid weight file, whose keys are torchvision's
(``Conv2d_1a_3x3.conv.weight``, ``Mixed_5b.branch_pool.bn.running_mean`` ...).  torch only holds the parameters: every conv, pool,
the resize and the fc run in csrc/inception_engine.cu.  No torchvision is needed, and nothing is ever downloaded."""
import ctypes as C
import os

import torch
from torch import nn

from .. import _native as N

# Inception weights ported to PyTorch from http://download.tensorflow.org/models/image/imagenet/inception-2015-12-05.tgz
FID_WEIGHTS_URL = 'https://github.com/mseitzer/pytorch-fid/releases/download/fid_weights/pt_inception-2015-12-05-6726825d.pth'  # noqa: E501
FID_WEIGHTS_FILE = os.path.basename(FID_WEIGHTS_URL)

RESIZE, NORMALIZE, OUT0, LOGITS = 1, 2, 4, 64     # rqb200_inception_forward flags (OUT<k> = OUT0 << k)
MIN_EXTENT = 75                                    # the smallest H, W the network takes without resizing (Mixed_7a)


class _Holder(nn.Module):
    def forward(self, *a, **k):
        raise RuntimeError("rqb200: parameter holder -- compute runs in the native engine (InceptionV3.forward)")


class BasicConv2d(_Holder):
    """torchvision's BasicConv2d: conv (no bias) + BatchNorm(eps 0.001) + ReLU"""
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_channels, eps=0.001)


class FIDInceptionA(_Holder):
    def __init__(self, in_channels, pool_features):
        super().__init__()
        self.branch1x1 = BasicConv2d(in_channels, 64, 1)
        self.branch5x5_1 = BasicConv2d(in_channels, 48, 1)
        self.branch5x5_2 = BasicConv2d(48, 64, 5, padding=2)
        self.branch3x3dbl_1 = BasicConv2d(in_channels, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, padding=1)
        self.branch_pool = BasicConv2d(in_channels, pool_features, 1)


class InceptionB(_Holder):
    def __init__(self, in_channels):
        super().__init__()
        self.branch3x3 = BasicConv2d(in_channels, 384, 3, stride=2)
        self.branch3x3dbl_1 = BasicConv2d(in_channels, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, stride=2)


class FIDInceptionC(_Holder):
    def __init__(self, in_channels, channels_7x7):
        super().__init__()
        c7 = channels_7x7
        self.branch1x1 = BasicConv2d(in_channels, 192, 1)
        self.branch7x7_1 = BasicConv2d(in_channels, c7, 1)
        self.branch7x7_2 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7_3 = BasicConv2d(c7, 192, (7, 1), padding=(3, 0))
        self.branch7x7dbl_1 = BasicConv2d(in_channels, c7, 1)
        self.branch7x7dbl_2 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_3 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7dbl_4 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_5 = BasicConv2d(c7, 192, (1, 7), padding=(0, 3))
        self.branch_pool = BasicConv2d(in_channels, 192, 1)


class InceptionD(_Holder):
    def __init__(self, in_channels):
        super().__init__()
        self.branch3x3_1 = BasicConv2d(in_channels, 192, 1)
        self.branch3x3_2 = BasicConv2d(192, 320, 3, stride=2)
        self.branch7x7x3_1 = BasicConv2d(in_channels, 192, 1)
        self.branch7x7x3_2 = BasicConv2d(192, 192, (1, 7), padding=(0, 3))
        self.branch7x7x3_3 = BasicConv2d(192, 192, (7, 1), padding=(3, 0))
        self.branch7x7x3_4 = BasicConv2d(192, 192, 3, stride=2)


class FIDInceptionE(_Holder):
    """FIDInceptionE_1 (average pool branch) and FIDInceptionE_2 (max pool branch) hold the same parameters"""
    def __init__(self, in_channels):
        super().__init__()
        self.branch1x1 = BasicConv2d(in_channels, 320, 1)
        self.branch3x3_1 = BasicConv2d(in_channels, 384, 1)
        self.branch3x3_2a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3_2b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch3x3dbl_1 = BasicConv2d(in_channels, 448, 1)
        self.branch3x3dbl_2 = BasicConv2d(448, 384, 3, padding=1)
        self.branch3x3dbl_3a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3dbl_3b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch_pool = BasicConv2d(in_channels, 192, 1)


class FIDInception3(_Holder):
    """the parameters of torchvision's Inception3(num_classes=1008, aux_logits=False) as patched by fid_inception_v3, under the
    torchvision names the pytorch-fid weight file uses"""
    def __init__(self):
        super().__init__()
        self.Conv2d_1a_3x3 = BasicConv2d(3, 32, 3, stride=2)
        self.Conv2d_2a_3x3 = BasicConv2d(32, 32, 3)
        self.Conv2d_2b_3x3 = BasicConv2d(32, 64, 3, padding=1)
        self.Conv2d_3b_1x1 = BasicConv2d(64, 80, 1)
        self.Conv2d_4a_3x3 = BasicConv2d(80, 192, 3)
        self.Mixed_5b = FIDInceptionA(192, pool_features=32)
        self.Mixed_5c = FIDInceptionA(256, pool_features=64)
        self.Mixed_5d = FIDInceptionA(288, pool_features=64)
        self.Mixed_6a = InceptionB(288)
        self.Mixed_6b = FIDInceptionC(768, channels_7x7=128)
        self.Mixed_6c = FIDInceptionC(768, channels_7x7=160)
        self.Mixed_6d = FIDInceptionC(768, channels_7x7=160)
        self.Mixed_6e = FIDInceptionC(768, channels_7x7=192)
        self.Mixed_7a = InceptionD(768)
        self.Mixed_7b = FIDInceptionE(1280)
        self.Mixed_7c = FIDInceptionE(2048)
        self.fc = nn.Linear(2048, 1008)


def fid_weights_path():
    """where the reference's load_state_dict_from_url caches the pytorch-fid weights: <torch.hub.get_dir()>/checkpoints/<file>
    (TORCH_HOME relocates it)"""
    return os.path.join(torch.hub.get_dir(), "checkpoints", FID_WEIGHTS_FILE)


def fid_inception_v3(path=None):
    """the FID Inception model with the pytorch-fid weights loaded from `path`, or from the torch hub cache where the reference and
    pytorch-fid put them.  Never downloads: a missing file raises FileNotFoundError naming the path looked at."""
    path = path or fid_weights_path()
    if not os.path.isfile(path):
        raise FileNotFoundError("rqb200: the FID Inception weights %s are not there.  This package never downloads; copy %s from "
                                "another machine's torch hub cache (or pass its path)" % (path, FID_WEIGHTS_URL))
    inception = FIDInception3()
    state_dict = torch.load(path, map_location="cpu", weights_only=True)
    inception.load_state_dict(state_dict)
    return inception


def block_extents(H, W, resize_input):
    """the (h, w) of blocks 0, 1, 2 for an H x W input"""
    if resize_input:
        H = W = 299

    def s2(n):                       # 3x3 stride-2 "valid" conv or max pool
        return (n - 3) // 2 + 1
    out = []
    h, w = s2(H) - 2, s2(W) - 2      # Conv2d_1a_3x3 (stride 2), Conv2d_2a_3x3; Conv2d_2b_3x3 keeps the extent
    h, w = s2(h), s2(w)              # max pool
    out.append((h, w))
    h, w = s2(h - 2), s2(w - 2)      # Conv2d_4a_3x3, max pool
    out.append((h, w))
    out.append((s2(h), s2(w)))       # Mixed_6a
    return out


class InceptionV3(N.EngineCache, nn.Module):
    """Pretrained InceptionV3 network returning feature maps (the reference's class; compute in the native engine).

    ``precision``: None (the default: RQB200_PRECISION, 'auto' = exact) or 'exact' run every conv on fp32 FFMA; 'fast' runs them (but
    the Cin = 3 Conv2d_1a_3x3) on the wgmma implicit GEMM with split-fp16 operands (three fp16 products per k step, fp32 accumulate)."""

    # Index of default block of inception to return, corresponds to output of final average pooling
    DEFAULT_BLOCK_INDEX = 3

    # Maps feature dimensionality to their output blocks indices
    BLOCK_INDEX_BY_DIM = {
        64: 0,   # First max pooling features
        192: 1,  # Second max pooling featurs
        768: 2,  # Pre-aux classifier features
        2048: 3  # Final average pooling features
    }
    BLOCK_CHANNELS = (64, 192, 768, 2048)

    def __init__(self, output_blocks=[DEFAULT_BLOCK_INDEX], resize_input=True, normalize_input=True, requires_grad=False,
                 use_fid_inception=True):
        super().__init__()
        self.resize_input = resize_input
        self.normalize_input = normalize_input
        self.output_blocks = sorted(output_blocks)
        self.last_needed_block = max(output_blocks)
        assert self.last_needed_block <= 3, 'Last possible output block index is 3'
        if not use_fid_inception:
            raise NotImplementedError("rqb200: use_fid_inception=False needs torchvision's ImageNet Inception weights, which this "
                                      "package does not load; FID uses the FID Inception (use_fid_inception=True)")
        self.blocks = nn.ModuleList()
        inception = fid_inception_v3()
        self.blocks.append(nn.Sequential(inception.Conv2d_1a_3x3, inception.Conv2d_2a_3x3, inception.Conv2d_2b_3x3,
                                         nn.MaxPool2d(kernel_size=3, stride=2)))
        if self.last_needed_block >= 1:
            self.blocks.append(nn.Sequential(inception.Conv2d_3b_1x1, inception.Conv2d_4a_3x3, nn.MaxPool2d(kernel_size=3, stride=2)))
        if self.last_needed_block >= 2:
            self.blocks.append(nn.Sequential(inception.Mixed_5b, inception.Mixed_5c, inception.Mixed_5d, inception.Mixed_6a,
                                             inception.Mixed_6b, inception.Mixed_6c, inception.Mixed_6d, inception.Mixed_6e))
        if self.last_needed_block >= 3:
            self.blocks.append(nn.Sequential(inception.Mixed_7a, inception.Mixed_7b, inception.Mixed_7c,
                                             nn.AdaptiveAvgPool2d(output_size=(1, 1))))
        self.fc = nn.Linear(2048, 1008, bias=True)
        with torch.no_grad():
            self.fc.weight.copy_(inception.fc.weight)
            self.fc.bias.copy_(inception.fc.bias)
        for param in self.parameters():
            param.requires_grad = requires_grad

    # ------------------------------------------------------------------ native engine plumbing
    _DESTROY = "rqb200_inception_destroy"

    def _engine(self, device):
        mode = self._mode()
        return self._cached_engine((str(device), mode), N.param_fingerprint(self), lambda: N.plan_engine(
            _lib(), "inception", IncConfig(self.last_needed_block, mode),
            {k: v for k, v in self.state_dict().items() if not k.endswith("num_batches_tracked")}, device))

    def _check_input(self, inp):
        if not isinstance(inp, torch.Tensor) or inp.dim() != 4:
            raise ValueError("InceptionV3: the input must be a 4-D [B, 3, H, W] tensor, got %s"
                             % (str(tuple(inp.shape)) if isinstance(inp, torch.Tensor) else type(inp).__name__))
        B, c, H, W = inp.shape
        if c != 3:
            raise ValueError("InceptionV3: the input has %d channels, the network takes 3 (shape %s)" % (c, tuple(inp.shape)))
        least = 1 if self.resize_input else MIN_EXTENT
        if B < 1 or H < least or W < least:
            raise ValueError("InceptionV3: need B >= 1 and H, W >= %d%s, got shape %s"
                             % (least, "" if self.resize_input else " without resize_input", tuple(inp.shape)))
        return B, H, W

    @torch.no_grad()
    def _run(self, inp, blocks, logits):
        """one native forward -> ({block: tensor}, logits or None)"""
        B, H, W = self._check_input(inp)
        if logits and self.last_needed_block != 3:
            raise ValueError("InceptionV3: return_logits needs the network through block 3 (output_blocks contains 3)")
        N.require_cuda(inp)
        x = inp.float().contiguous()
        eng = self._engine(x.device)
        L = _lib()
        flags = (RESIZE if self.resize_input else 0) | (NORMALIZE if self.normalize_input else 0) | (LOGITS if logits else 0)
        ext = block_extents(H, W, self.resize_input)
        outs = [None] * 4
        for k in blocks:
            flags |= OUT0 << k
            shape = (B, 2048, 1, 1) if k == 3 else (B, self.BLOCK_CHANNELS[k]) + ext[k]
            outs[k] = torch.empty(shape, dtype=torch.float32, device=x.device)
        lg = torch.empty(B, 1008, dtype=torch.float32, device=x.device) if logits else None
        with torch.cuda.device(x.device):
            ws = N.workspace(eng, L.rqb200_inception_workspace_bytes(eng["handle"], B, H, W, flags), x.device,
                             "rqb200_inception_workspace_bytes: extent %d x %d refused" % (H, W))
            N.check(L.rqb200_inception_forward(eng["handle"], N.ptr(x), B, H, W, flags, *[N.ptr(o) for o in outs], N.ptr(lg), N.ptr(ws),
                                               ws.numel(), N.stream_ptr(x.device)), "inception_forward")
        self.last_launches = L.rqb200_inception_last_launches(eng["handle"])
        N.launch_count["total"] += self.last_launches
        return outs, lg

    def forward(self, inp, return_logits=False):
        """Get Inception feature maps.  inp [B, 3, H, W] in (0, 1) on a CUDA device; returns the list of the selected blocks' outputs,
        sorted ascending by index (block 3: [B, 2048, 1, 1]), and with return_logits the [B, 1008] fc logits as well."""
        outs, lg = self._run(inp, self.output_blocks, return_logits)
        outp = [outs[k] for k in self.output_blocks]
        if return_logits:
            return outp, lg
        return outp


class IncConfig(C.Structure):
    _fields_ = [("last_block", C.c_int32), ("mode", C.c_int32)]


def _lib():
    L = N.lib()
    if not getattr(L, "_inception_bound", False):
        N.bind_plan_engine(L, "inception", IncConfig)
        L.rqb200_inception_workspace_bytes.restype = C.c_size_t
        L.rqb200_inception_workspace_bytes.argtypes = [C.c_void_p] + [C.c_int] * 4
        L.rqb200_inception_forward.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p] * 6 + [C.c_size_t, C.c_void_p]
        L.rqb200_dbg_inception_conv.argtypes = [C.c_void_p] * 4 + [C.c_int] * 12 + [C.c_void_p]
        L.rqb200_dbg_inception_conv_tc.argtypes = [C.c_void_p] * 8 + [C.c_int] * 12 + [C.c_void_p]
        L.rqb200_dbg_inception_input.argtypes = [C.c_void_p] * 2 + [C.c_int] * 5 + [C.c_void_p]
        L.rqb200_dbg_inception_pool.argtypes = [C.c_int] + [C.c_void_p] * 2 + [C.c_int] * 8 + [C.c_void_p]
        L.rqb200_dbg_inception_gap.argtypes = [C.c_void_p] * 2 + [C.c_int] * 3 + [C.c_void_p]
        L._inception_bound = True
    return L


EXPORTS = [n for n in N.EXPORTS if "inception" in n]       # the C exports this module binds
