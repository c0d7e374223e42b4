"""LPIPS -- host-side mirror of rqvae/losses/vqgan/lpips.py (the VGG16 learned perceptual metric) over the native LPIPS engine.

Boundary kept: ``LPIPS(use_dropout=True)``, ``forward(input, target, reduction='mean')``, ``load_from_pretrained`` /
``from_pretrained``, ``ScalingLayer``, ``NetLinLayer``, ``vgg16``, ``normalize_tensor``, ``spatial_average`` and the state_dict key
layout (``scaling_layer.shift`` ... ``net.slice5.28.bias``, ``lin{k}.model.1.weight`` with dropout, ``lin{k}.model.0.weight`` without).
torch only holds the parameters: the scaling, the 13 VGG convs, the pools and the heads run in csrc/lpips_engine.cu, forward only.
No torchvision is needed, and nothing is ever downloaded.

Deviation: the reference broadcasts a batch-1 target against a larger input; here input and target must have equal shapes."""
import ctypes as C
import os

import torch
from torch import nn

from ... import _native as N
from .lpips_utils import get_ckpt_path, vgg16_weights_path, VGG16_URL

MIN_EXTENT = 16                                  # four 2x2 pools must leave relu5_3 at least 1 x 1
REDUCTIONS = ("none", "mean", "sum")
# vgg16.features[:30] by slice: (index, Cout) of each conv; a ReLU follows every conv, a 2x2 max pool opens slices 2..5
VGG_SLICES = (((0, 64), (2, 64)), ((5, 128), (7, 128)), ((10, 256), (12, 256), (14, 256)), ((17, 512), (19, 512), (21, 512)),
              ((24, 512), (26, 512), (28, 512)))


class LPIPS(N.EngineCache, nn.Module):
    """Learned perceptual metric (the reference's class; compute in the native engine, forward only).

    ``precision``: None (the default: RQB200_PRECISION, 'auto' = exact) or 'exact' run every conv on fp32 FFMA; 'fast' runs them (but the
    Cin = 3 conv1_1) on the wgmma implicit GEMM with split-fp16 operands (three fp16 products per k step, fp32 accumulate)."""

    def __init__(self, use_dropout=True):
        super().__init__()
        self.scaling_layer = ScalingLayer()
        self.chns = [64, 128, 256, 512, 512]  # vg16 features
        self.net = vgg16(pretrained=True, requires_grad=False)
        self.lin0 = NetLinLayer(self.chns[0], use_dropout=use_dropout)
        self.lin1 = NetLinLayer(self.chns[1], use_dropout=use_dropout)
        self.lin2 = NetLinLayer(self.chns[2], use_dropout=use_dropout)
        self.lin3 = NetLinLayer(self.chns[3], use_dropout=use_dropout)
        self.lin4 = NetLinLayer(self.chns[4], use_dropout=use_dropout)
        self.use_dropout = use_dropout
        self.load_from_pretrained()
        for param in self.parameters():
            param.requires_grad = False

    def load_from_pretrained(self, name="vgg_lpips"):
        ckpt = get_ckpt_path(name)
        self.load_state_dict(torch.load(ckpt, map_location=torch.device("cpu"), weights_only=True), strict=False)
        print("loaded pretrained LPIPS loss from {}".format(ckpt))

    @classmethod
    def from_pretrained(cls, name="vgg_lpips"):
        if name != "vgg_lpips":
            raise NotImplementedError
        model = cls()
        ckpt = get_ckpt_path(name)
        model.load_state_dict(torch.load(ckpt, map_location=torch.device("cpu"), weights_only=True), strict=False)
        return model

    # ------------------------------------------------------------------ native engine plumbing
    _DESTROY = "rqb200_lpips_destroy"

    def _engine(self, device):
        mode = self._mode()
        return self._cached_engine((str(device), mode), N.param_fingerprint(self),
                                   lambda: N.plan_engine(_lib(), "lpips", LpipsConfig(mode), self.state_dict(), device))

    def _check(self, input, target, reduction):
        for name, t in (("input", input), ("target", target)):
            if not isinstance(t, torch.Tensor) or t.dim() != 4:
                raise ValueError("LPIPS: the %s must be a 4-D [B, 3, H, W] tensor, got %s"
                                 % (name, str(tuple(t.shape)) if isinstance(t, torch.Tensor) else type(t).__name__))
            if t.shape[1] != 3:
                raise ValueError("LPIPS: the %s has %d channels, the network takes 3 (shape %s)" % (name, t.shape[1], tuple(t.shape)))
        if input.shape != target.shape:
            raise ValueError("LPIPS: input %s and target %s must have the same shape (a batch-1 target is not broadcast)"
                             % (tuple(input.shape), tuple(target.shape)))
        B, _, H, W = input.shape
        if B < 1 or H < MIN_EXTENT or W < MIN_EXTENT:
            raise ValueError("LPIPS: need B >= 1 and H, W >= %d (four 2x2 pools leave relu5_3 at least 1 x 1), got shape %s"
                             % (MIN_EXTENT, tuple(input.shape)))
        if reduction not in REDUCTIONS:
            raise ValueError("LPIPS: reduction must be one of %s, got %r" % (", ".join(REDUCTIONS), reduction))
        if not input.is_cuda or input.device != target.device:
            raise ValueError("LPIPS: input and target must be on one CUDA device, got %s and %s" % (input.device, target.device))
        if self.training and self.use_dropout:
            raise NotImplementedError("rqb200: LPIPS in training mode would apply dropout, which is out of scope; call .eval()")
        if torch.is_grad_enabled() and (input.requires_grad or target.requires_grad):
            raise RuntimeError("rqb200: LPIPS has no backward; call it under torch.no_grad() or on tensors that do not require grad")
        return B, H, W

    def _run(self, input, target, reduction="none"):
        """one native forward -> (per-tap spatial averages [B, 5], values [B]) as float32"""
        B, H, W = self._check(input, target, reduction)
        x0 = input.detach().float().contiguous()
        x1 = target.detach().float().contiguous()
        eng = self._engine(x0.device)
        L = _lib()
        layers = torch.empty(B, 5, dtype=torch.float32, device=x0.device)
        val = torch.empty(B, dtype=torch.float32, device=x0.device)
        with torch.cuda.device(x0.device):
            ws = N.workspace(eng, L.rqb200_lpips_workspace_bytes(eng["handle"], B, H, W), x0.device,
                             "rqb200_lpips_workspace_bytes: extent %d x %d refused" % (H, W))
            N.check(L.rqb200_lpips_forward(eng["handle"], N.ptr(x0), N.ptr(x1), B, H, W, N.ptr(layers), N.ptr(val), N.ptr(ws), ws.numel(),
                                           N.stream_ptr(x0.device)), "lpips_forward")
        self.last_launches = L.rqb200_lpips_last_launches(eng["handle"])
        N.launch_count["total"] += self.last_launches
        return layers, val

    def forward(self, input, target, reduction='mean'):
        """input, target [B, 3, H, W] in [-1, 1] on one CUDA device, equal shapes, H, W >= 16.  reduction 'none' -> [B, 1, 1, 1];
        'mean' / 'sum' -> a scalar."""
        _, val = self._run(input, target, reduction)
        val = val.reshape(-1, 1, 1, 1)
        if reduction == 'none':
            return val
        elif reduction == 'mean':
            return torch.mean(val)
        return torch.sum(val)


class ScalingLayer(nn.Module):
    def __init__(self):
        super(ScalingLayer, self).__init__()
        self.register_buffer('shift', torch.Tensor([-.030, -.088, -.188])[None, :, None, None])
        self.register_buffer('scale', torch.Tensor([.458, .448, .450])[None, :, None, None])

    def forward(self, inp):
        return (inp - self.shift) / self.scale


class NetLinLayer(nn.Module):
    """ A single linear layer which does a 1x1 conv """
    def __init__(self, chn_in, chn_out=1, use_dropout=False):
        super(NetLinLayer, self).__init__()
        layers = [nn.Dropout(), ] if (use_dropout) else []
        layers += [nn.Conv2d(chn_in, chn_out, 1, stride=1, padding=0, bias=False), ]
        self.model = nn.Sequential(*layers)


def vgg16_features_weights(path=None):
    """the conv weights of torchvision's ImageNet VGG16 (features.<i>.weight / .bias of features[:30]) from `path`, or from the torch
    hub cache where models.vgg16(pretrained=True) puts them.  Never downloads: a missing file raises FileNotFoundError naming the path."""
    path = path or vgg16_weights_path()
    if not os.path.isfile(path):
        raise FileNotFoundError("rqb200: the VGG16 weights %s are not there.  This package never downloads; copy %s from another "
                                "machine's torch hub cache (or pass its path)" % (path, VGG16_URL))
    sd = torch.load(path, map_location="cpu", weights_only=True)
    return {k: v for k, v in sd.items() if k.startswith("features.") and int(k.split(".")[1]) < 30}


class vgg16(nn.Module):
    """torchvision's VGG16 features[:30] in the reference's five slices (the same module indices, so the same state_dict keys).  A
    parameter holder: its convs run in the native engine (LPIPS.forward).  pretrained=False keeps torch's default initialisation."""
    def __init__(self, requires_grad=False, pretrained=True):
        super(vgg16, self).__init__()
        cin = 3
        for s, convs in enumerate(VGG_SLICES):
            sl = nn.Sequential()
            if s > 0:
                sl.add_module(str(convs[0][0] - 1), nn.MaxPool2d(kernel_size=2, stride=2, padding=0, dilation=1, ceil_mode=False))
            for i, cout in convs:
                sl.add_module(str(i), nn.Conv2d(cin, cout, kernel_size=3, padding=1))
                sl.add_module(str(i + 1), nn.ReLU(inplace=True))
                cin = cout
            setattr(self, "slice%d" % (s + 1), sl)
        self.N_slices = 5
        if pretrained:
            sd = vgg16_features_weights()
            with torch.no_grad():
                for s, convs in enumerate(VGG_SLICES):
                    sl = getattr(self, "slice%d" % (s + 1))
                    for i, _ in convs:
                        getattr(sl, str(i)).weight.copy_(sd["features.%d.weight" % i])
                        getattr(sl, str(i)).bias.copy_(sd["features.%d.bias" % i])
        if not requires_grad:
            for param in self.parameters():
                param.requires_grad = False

    def forward(self, X):
        raise RuntimeError("rqb200: parameter holder -- the VGG16 runs in the native engine (LPIPS.forward)")


def normalize_tensor(x, eps=1e-10):
    norm_factor = torch.sqrt(torch.sum(x**2, dim=1, keepdim=True))
    return x/(norm_factor+eps)


def spatial_average(x, keepdim=True):
    return x.mean([2, 3], keepdim=keepdim)


class LpipsConfig(C.Structure):
    _fields_ = [("mode", C.c_int32)]


def _lib():
    L = N.lib()
    if not getattr(L, "_lpips_bound", False):
        N.bind_plan_engine(L, "lpips", LpipsConfig)
        L.rqb200_lpips_workspace_bytes.restype = C.c_size_t
        L.rqb200_lpips_workspace_bytes.argtypes = [C.c_void_p] + [C.c_int] * 3
        L.rqb200_lpips_forward.argtypes = [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p] * 3 + [C.c_size_t, C.c_void_p]
        L.rqb200_dbg_lpips_input.argtypes = [C.c_void_p] * 5 + [C.c_int] * 3 + [C.c_void_p]
        L.rqb200_dbg_lpips_pool.argtypes = [C.c_void_p] * 4 + [C.c_int] * 4 + [C.c_void_p]
        L.rqb200_dbg_lpips_head.argtypes = [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p]
        L.rqb200_dbg_lpips_mean.argtypes = [C.c_void_p] + [C.c_int] * 3 + [C.c_void_p] * 4
        L._lpips_bound = True
    return L


EXPORTS = [n for n in N.EXPORTS if "lpips" in n]       # the C exports this module binds
