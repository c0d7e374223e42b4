"""TEST INFRASTRUCTURE ONLY -- a float64 restatement of torchvision's resnet101 forward (the v1.5 Bottleneck, eval-mode BatchNorm) and
its IMAGENET1K_V1 eval preprocessing without the resize (CenterCrop, Normalize), with no torchvision import; plus the seeded synthetic
weights and inputs of tests/golden/resnet.pt (scripts/gen_golden_resnet.py), which pins this restatement to torchvision."""
import torch
import torch.nn.functional as F

LAYERS = (3, 4, 23, 3)
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
BN_EPS = 1e-5
# the last BatchNorm of each block scales its branch by about this much, so the residual stream stays O(1) through 33 adds
BRANCH_GAIN = 0.12


def convs():
    """(conv key, bn key, Cin, Cout, k) of every conv in torchvision's state_dict order"""
    out = [("conv1", "bn1", 3, 64, 7)]
    cin = 64
    for i, n in enumerate(LAYERS):
        w = 64 << i
        for b in range(n):
            p = "layer%d.%d." % (i + 1, b)
            out += [(p + "conv1", p + "bn1", cin, w, 1), (p + "conv2", p + "bn2", w, w, 3), (p + "conv3", p + "bn3", w, 4 * w, 1)]
            if b == 0:
                out.append((p + "downsample.0", p + "downsample.1", cin, 4 * w, 1))
            cin = 4 * w
    return out


def state_dict_shapes():
    """{key: shape} of torchvision's resnet101().state_dict(), in its order"""
    sh = {}
    for conv, bn, ci, co, k in convs():
        sh[conv + ".weight"] = (co, ci, k, k)
        for s in ("weight", "bias", "running_mean", "running_var"):
            sh[bn + "." + s] = (co,)
        sh[bn + ".num_batches_tracked"] = ()
    sh["fc.weight"] = (1000, 2048)
    sh["fc.bias"] = (1000,)
    return sh


def synth_weights(seed):
    """seeded fp32 weights that keep activations O(1): He-scaled convs, BatchNorm statistics near the identity, each block's bn3 scale
    multiplied by BRANCH_GAIN, and an fc whose logits spread over a few units"""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for conv, bn, ci, co, k in convs():
        sd[conv + ".weight"] = torch.randn(co, ci, k, k, generator=g) * (2.0 / (ci * k * k)) ** 0.5
        gain = BRANCH_GAIN if bn.endswith("bn3") else 1.0
        sd[bn + ".weight"] = (0.75 + 0.5 * torch.rand(co, generator=g)) * gain
        sd[bn + ".bias"] = 0.05 * torch.randn(co, generator=g)
        sd[bn + ".running_mean"] = 0.05 * torch.randn(co, generator=g)
        sd[bn + ".running_var"] = 0.8 + 0.45 * torch.rand(co, generator=g)
        sd[bn + ".num_batches_tracked"] = torch.tensor(0)
    sd["fc.weight"] = torch.randn(1000, 2048, generator=g) * (0.25 / 2048) ** 0.5
    sd["fc.bias"] = 0.1 * torch.randn(1000, generator=g)
    return {k: sd[k] for k in state_dict_shapes()}


def case_inputs(case):
    """the fp32 pixels in [0, 1] of a fixture case"""
    g = torch.Generator().manual_seed(case["seed"])
    return torch.rand(case["B"], 3, case["H"], case["W"], generator=g)


def crop_offset(n, c):
    return int(round((n - c) / 2.0))                 # torchvision CenterCrop


def preprocess(x, center_crop=224):
    """CenterCrop(center_crop) (None: the whole image) and Normalize, in x's dtype"""
    if center_crop is not None:
        t, l = crop_offset(x.shape[2], center_crop), crop_offset(x.shape[3], center_crop)
        x = x[:, :, t:t + center_crop, l:l + center_crop]
    mean = torch.tensor(MEAN, dtype=x.dtype, device=x.device).reshape(1, 3, 1, 1)
    std = torch.tensor(STD, dtype=x.dtype, device=x.device).reshape(1, 3, 1, 1)
    return (x - mean) / std


def _cbn(sd, x, conv, bn, stride, pad):
    x = F.conv2d(x, sd[conv + ".weight"], None, stride, pad)
    return F.batch_norm(x, sd[bn + ".running_mean"], sd[bn + ".running_var"], sd[bn + ".weight"], sd[bn + ".bias"], False, 0.0, BN_EPS)


def features(sd, x):
    """the pooled features [B, 2048] of preprocessed x [B, 3, H, W] (sd in x's dtype and device)"""
    x = F.relu(_cbn(sd, x, "conv1", "bn1", 2, 3))
    x = F.max_pool2d(x, 3, 2, 1)
    for i, n in enumerate(LAYERS):
        for b in range(n):
            p = "layer%d.%d." % (i + 1, b)
            s = 2 if (b == 0 and i > 0) else 1
            o = F.relu(_cbn(sd, x, p + "conv1", p + "bn1", 1, 0))
            o = F.relu(_cbn(sd, o, p + "conv2", p + "bn2", s, 1))
            o = _cbn(sd, o, p + "conv3", p + "bn3", 1, 0)
            idn = _cbn(sd, x, p + "downsample.0", p + "downsample.1", s, 0) if b == 0 else x
            x = F.relu(o + idn)
    return x.mean((2, 3))


def logits(sd, x, center_crop=224):
    """torchvision's resnet101(x') with x' = preprocess(x): logits [B, 1000] in x's dtype"""
    f = features(sd, preprocess(x, center_crop))
    return F.linear(f, sd["fc.weight"], sd["fc.bias"])


def sd_as(sd, dtype=torch.float64, device="cpu"):
    return {k: (v.to(device=device, dtype=dtype) if v.is_floating_point() else v.to(device)) for k, v in sd.items()}
