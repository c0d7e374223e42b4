"""ResNet-101 -- torchvision's ImageNet classifier (models.resnet101, IMAGENET1K_V1 weights) over the native ResNet engine, forward only.

It scores class-conditional samples: ``class_log_prob`` gives each image's log-probability of its requested class, which is what
rejection sampling (rqvae.models.rqtransformer.rejection_sample) keeps the best candidate by, and a per-batch check of class-conditional
sampling on its own.  torch only holds the parameters, under torchvision's state_dict keys, so torchvision's weight file loads strictly;
the crop, the normalisation, the 104 convs, the pools and fc run in csrc/resnet_engine.cu.  No torchvision is needed, and nothing is
ever downloaded.

Preprocessing: torchvision's IMAGENET1K_V1 eval transform is Resize(256), CenterCrop(224), Normalize(ImageNet mean, std).  For a 256^2
image Resize(256) is the identity, so ``forward(pixels)`` with the default ``center_crop=224`` IS that transform.  Deviation: no resize
is done at other sizes; a caller whose smaller side is not 256 resizes first (or passes ``center_crop=None`` to classify the whole
image)."""
import ctypes as C
import os

import torch
from torch import nn

from .. import _native as N

MIN_EXTENT = 32                  # the smallest H, W (after the crop) the engine takes: layer4 sees 1 x 1
NUM_CLASSES = 1000
FEATURES = 2048
LAYERS = (3, 4, 23, 3)           # Bottleneck blocks per stage
RESNET101_URL = "https://download.pytorch.org/models/resnet101-63fe2227.pth"   # models.ResNet101_Weights.IMAGENET1K_V1
RESNET101_FILE = os.path.basename(RESNET101_URL)
FLAG_FEATURES = 1


def resnet101_weights_path():
    """where models.resnet101(weights=IMAGENET1K_V1) caches torchvision's weights: <torch.hub.get_dir()>/checkpoints/<file>"""
    return os.path.join(torch.hub.get_dir(), "checkpoints", RESNET101_FILE)


class Bottleneck(nn.Module):
    """torchvision's v1.5 Bottleneck (the stride on the 3x3), as a parameter holder"""
    expansion = 4

    def __init__(self, inplanes, width, stride=1, downsample=False):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, width, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, 3, stride=stride, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, width * 4, 1, bias=False)
        self.bn3 = nn.BatchNorm2d(width * 4)
        self.relu = nn.ReLU(inplace=True)
        self.downsample = nn.Sequential(nn.Conv2d(inplanes, width * 4, 1, stride=stride, bias=False),
                                        nn.BatchNorm2d(width * 4)) if downsample else None
        self.stride = stride


class ResNet101(N.EngineCache, nn.Module):
    """torchvision's resnet101 with its parameter and buffer names; the forward runs in the native engine.

    ``precision``: None (the default: RQB200_PRECISION, 'auto' = exact) or 'exact' run every conv on fp32 FFMA; 'fast' runs them (but the
    Cin = 3 stem conv) on the wgmma implicit GEMM with split-fp16 operands (three fp16 products per k step, fp32 accumulate).  The
    residual stream and fc are fp32 on both tiers.  The engine is rebuilt when the parameters change."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.relu = nn.ReLU(inplace=True)
        self.maxpool = nn.MaxPool2d(kernel_size=3, stride=2, padding=1)
        inplanes = 64
        for i, n in enumerate(LAYERS):
            width = 64 << i
            blocks = [Bottleneck(inplanes, width, 1 if i == 0 else 2, True)] + [Bottleneck(width * 4, width) for _ in range(n - 1)]
            setattr(self, "layer%d" % (i + 1), nn.Sequential(*blocks))
            inplanes = width * 4
        self.avgpool = nn.AdaptiveAvgPool2d((1, 1))
        self.fc = nn.Linear(FEATURES, NUM_CLASSES)
        for p in self.parameters():
            p.requires_grad = False
        self.eval()

    # ------------------------------------------------------------------ native engine plumbing
    _DESTROY = "rqb200_resnet_destroy"

    def _engine(self, device):
        mode = self._mode()
        return self._cached_engine((str(device), mode), N.param_fingerprint(self),
                                   lambda: N.plan_engine(_lib(), "resnet", ResnetConfig(mode), self.state_dict(), device))

    @staticmethod
    def _check(pixels, center_crop, device=True):
        if not isinstance(pixels, torch.Tensor) or pixels.dim() != 4:
            raise ValueError("ResNet101: pixels must be a 4-D [B, 3, H, W] tensor, got %s"
                             % (str(tuple(pixels.shape)) if isinstance(pixels, torch.Tensor) else type(pixels).__name__))
        B, ch, H, W = pixels.shape
        if ch != 3:
            raise ValueError("ResNet101: pixels have %d channels, the network takes 3 (shape %s)" % (ch, tuple(pixels.shape)))
        if B < 1:
            raise ValueError("ResNet101: empty batch")
        if center_crop is not None:
            if isinstance(center_crop, bool) or not isinstance(center_crop, int) or center_crop < MIN_EXTENT:
                raise ValueError("ResNet101: center_crop must be None or an int >= %d, got %r" % (MIN_EXTENT, center_crop))
            if H < center_crop or W < center_crop:
                raise ValueError("ResNet101: a %d x %d image is smaller than center_crop=%d (no resize is done; resize first)"
                                 % (H, W, center_crop))
        elif H < MIN_EXTENT or W < MIN_EXTENT:
            raise ValueError("ResNet101: need H, W >= %d, got %d x %d" % (MIN_EXTENT, H, W))
        if device and not pixels.is_cuda:
            raise ValueError("ResNet101: pixels on %s; the engine runs on CUDA only" % pixels.device)
        if torch.is_grad_enabled() and pixels.requires_grad:
            raise RuntimeError("rqb200: ResNet101 has no backward; call it under torch.no_grad() or on tensors that do not require grad")
        return B, H, W

    def _run(self, pixels, center_crop=224, features=False):
        """one native forward -> logits [B, 1000] (and the pooled features [B, 2048] when features) as float32"""
        B, H, W = self._check(pixels, center_crop)
        x = pixels.detach().float().contiguous()
        eng = self._engine(x.device)
        L = _lib()
        flags = (center_crop or 0) << 8 | (FLAG_FEATURES if features else 0)
        logits = torch.empty(B, NUM_CLASSES, dtype=torch.float32, device=x.device)
        feat = torch.empty(B, FEATURES, dtype=torch.float32, device=x.device) if features else None
        with torch.cuda.device(x.device):
            ws = N.workspace(eng, L.rqb200_resnet_workspace_bytes(eng["handle"], B, H, W, flags), x.device,
                             "rqb200_resnet_workspace_bytes: extent %d x %d refused" % (H, W))
            N.check(L.rqb200_resnet_forward(eng["handle"], N.ptr(x), B, H, W, flags, N.ptr(logits), N.ptr(feat), N.ptr(ws), ws.numel(),
                                            N.stream_ptr(x.device)), "resnet_forward")
        self.last_launches = L.rqb200_resnet_last_launches(eng["handle"])
        N.launch_count["total"] += self.last_launches
        return (logits, feat) if features else logits

    def forward(self, pixels, center_crop=224):
        """pixels [B, 3, H, W] fp32 in [0, 1] on CUDA -> logits [B, 1000].  center_crop: the side of the centre window classified
        (torchvision CenterCrop's offsets), or None for the whole image; H, W >= 32."""
        return self._run(pixels, center_crop)

    def class_log_prob(self, pixels, labels, center_crop=224):
        """log_softmax(logits)[b, labels[b]] as fp32 [B]; labels: integer [B] in [0, 1000)"""
        B = self._check(pixels, center_crop, device=False)[0]
        if not isinstance(labels, torch.Tensor) or labels.dtype.is_floating_point or labels.dtype.is_complex or \
                labels.dtype == torch.bool or labels.dim() != 1 or labels.shape[0] != B:
            raise ValueError("ResNet101: labels must be an integer [B] tensor (B = %s), got %s %s"
                             % (B, getattr(labels, "dtype", type(labels).__name__), tuple(getattr(labels, "shape", ()))))
        if labels.numel() and (int(labels.min()) < 0 or int(labels.max()) >= NUM_CLASSES):
            raise ValueError("ResNet101: labels must lie in [0, %d)" % NUM_CLASSES)
        logits = self._run(pixels, center_crop)
        idx = labels.to(device=logits.device, dtype=torch.int64)
        return torch.log_softmax(logits, dim=1).gather(1, idx[:, None])[:, 0]


def get_resnet101(path=None):
    """ResNet101 with torchvision's IMAGENET1K_V1 weights from `path`, or from the torch hub cache where models.resnet101(weights=
    IMAGENET1K_V1) puts them (resnet101_weights_path()); any torchvision ResNet-101 state_dict file loads.  Never downloads: a missing
    file raises FileNotFoundError naming the path looked at."""
    path = path or resnet101_weights_path()
    if not os.path.isfile(path):
        raise FileNotFoundError("rqb200: the ResNet-101 weights %s are not there.  This package never downloads; copy %s from another "
                                "machine's torch hub cache (or pass its path)" % (path, RESNET101_URL))
    model = ResNet101()
    model.load_state_dict(torch.load(path, map_location="cpu", weights_only=True))
    return model


class ResnetConfig(C.Structure):
    _fields_ = [("mode", C.c_int32)]


def _lib():
    L = N.lib()
    if not getattr(L, "_resnet_bound", False):
        N.bind_plan_engine(L, "resnet", ResnetConfig)
        L.rqb200_resnet_workspace_bytes.restype = C.c_size_t
        L.rqb200_resnet_workspace_bytes.argtypes = [C.c_void_p] + [C.c_int] * 4
        L.rqb200_resnet_forward.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 4 + [C.c_void_p] * 3 + [C.c_size_t, C.c_void_p]
        L.rqb200_dbg_resnet_input.argtypes = [C.c_void_p] * 2 + [C.c_int] * 4 + [C.c_void_p]
        L.rqb200_dbg_resnet_conv.argtypes = [C.c_void_p] * 5 + [C.c_int] * 11 + [C.c_void_p]
        L.rqb200_dbg_resnet_conv_tc.argtypes = [C.c_void_p] * 9 + [C.c_int] * 11 + [C.c_void_p]
        L._resnet_bound = True
    return L


EXPORTS = [n for n in N.EXPORTS if "resnet" in n]       # the C exports this module binds
