"""TEST INFRASTRUCTURE ONLY -- a torch restatement of LPIPS (rqvae/losses/vqgan/lpips.py over torchvision's VGG16 features[:30]) on
the reference's LPIPS state_dict layout (``scaling_layer.*``, ``net.slice<s>.<i>.*``, ``lin<k>.model.<j>.weight``).

F.conv2d + F.relu, F.max_pool2d(2, 2), normalize_tensor, the squared difference, the 1x1 lin conv and the spatial mean, in whatever
dtype the state_dict and inputs come in (float64 for the fixture comparisons).  Pinned to tests/golden/lpips.pt
(tests/test_host_lpips.py); the GPU tests use it at sizes and batches the fixture does not hold.  Also builds the fixture's synthetic
weights from its seed and writes them where rqvae.losses.vqgan.lpips looks for them."""
import os

import torch
import torch.nn.functional as F

from oracle import synth

CHNS = (64, 128, 256, 512, 512)
# (state_dict prefix, Cin, Cout, tap): the 13 convs of vgg16.features[:30]; a 2x2 max pool follows every tap but the last
CONVS = [("net.slice1.0", 3, 64, False), ("net.slice1.2", 64, 64, True),
         ("net.slice2.5", 64, 128, False), ("net.slice2.7", 128, 128, True),
         ("net.slice3.10", 128, 256, False), ("net.slice3.12", 256, 256, False), ("net.slice3.14", 256, 256, True),
         ("net.slice4.17", 256, 512, False), ("net.slice4.19", 512, 512, False), ("net.slice4.21", 512, 512, True),
         ("net.slice5.24", 512, 512, False), ("net.slice5.26", 512, 512, False), ("net.slice5.28", 512, 512, True)]
SHIFT = [-.030, -.088, -.188]
SCALE = [.458, .448, .450]
VGG16_FILE = "vgg16-397923af.pth"


def synth_weights(seed, use_dropout=True):
    """the fixture's synthetic LPIPS state_dict (float32): He-scaled VGG convs, so every tap stays O(1) through 13 ReLU convs; small
    biases; non-negative lin weights, like the trained ones"""
    sd = {"scaling_layer.shift": torch.tensor(SHIFT).reshape(1, 3, 1, 1), "scaling_layer.scale": torch.tensor(SCALE).reshape(1, 3, 1, 1)}
    for i, (name, ci, co, _) in enumerate(CONVS):
        sd[name + ".weight"] = synth.randn_seeded((co, ci, 3, 3), seed + 2 * i, (2.0 / (9 * ci)) ** 0.5)
        sd[name + ".bias"] = synth.randn_seeded((co,), seed + 2 * i + 1, 0.01)
    j = 1 if use_dropout else 0
    for k, c in enumerate(CHNS):
        sd["lin%d.model.%d.weight" % (k, j)] = synth.randn_seeded((1, c, 1, 1), seed + 100 + k, 0.1).abs()
    return sd


def write_weight_files(torch_home, sd):
    """sd (use_dropout=True layout) as the two files rqvae.losses.vqgan.lpips reads under TORCH_HOME = torch_home: torchvision's
    VGG16 (features.<i>.* keys) and the LPIPS vgg.pth (lin<k>.model.1.weight, as the published file).  Returns their paths."""
    d = os.path.join(torch_home, "hub", "checkpoints")
    os.makedirs(d, exist_ok=True)
    vgg = {"features." + k.split(".", 2)[2]: v for k, v in sd.items() if k.startswith("net.")}
    lin = {k: v for k, v in sd.items() if k.startswith("lin")}
    p1, p2 = os.path.join(d, VGG16_FILE), os.path.join(d, "vgg.pth")
    torch.save(vgg, p1)
    torch.save(lin, p2)
    return p1, p2


def lin_weight(sd, k):
    w = sd.get("lin%d.model.1.weight" % k)
    return w if w is not None else sd["lin%d.model.0.weight" % k]


def features(sd, x):
    """the five taps relu1_2 .. relu5_3 of the scaled input x [B, 3, H, W]"""
    shift = sd["scaling_layer.shift"].to(x)
    scale = sd["scaling_layer.scale"].to(x)
    h = (x - shift) / scale
    taps = []
    for name, _, _, tap in CONVS:
        h = F.relu(F.conv2d(h, sd[name + ".weight"].to(x), sd[name + ".bias"].to(x), padding=1))
        if tap:
            taps.append(h)
            if len(taps) < len(CHNS):
                h = F.max_pool2d(h, 2, 2)
    return taps


def normalize_tensor(x, eps=1e-10):
    return x / (torch.sqrt(torch.sum(x ** 2, dim=1, keepdim=True)) + eps)


def lpips(sd, x0, x1):
    """-> (per-tap spatial averages [B, 5], values [B]) of the pairs (x0[b], x1[b])"""
    f0, f1 = features(sd, x0), features(sd, x1)
    layers = []
    for k in range(len(CHNS)):
        d = (normalize_tensor(f0[k]) - normalize_tensor(f1[k])) ** 2
        layers.append(F.conv2d(d, lin_weight(sd, k).to(d)).mean([2, 3]).reshape(-1))
    layers = torch.stack(layers, 1)
    return layers, layers.sum(1)


def case_inputs(case):
    """the fixture case's (input, target) float32 pair in [-1, 1]: seeded uniform; 'identical' target = input; 'noisy' target = input
    + 0.01 N(0, 1) (a reconstruction-like pair)"""
    g = torch.Generator().manual_seed(case["seed"])
    shape = (case["B"], 3, case["H"], case["W"])
    x0 = torch.rand(shape, generator=g) * 2 - 1
    if case["kind"] == "identical":
        return x0, x0.clone()
    if case["kind"] == "noisy":
        return x0, x0 + 0.01 * torch.randn(shape, generator=g)
    return x0, torch.rand(shape, generator=g) * 2 - 1
