"""TEST INFRASTRUCTURE ONLY -- a torch restatement of the FID Inception-v3 (rqvae/metrics/inception.py over torchvision's
Inception3 as patched by fid_inception_v3) on the reference's InceptionV3 state_dict layout (``blocks.*``, ``fc.*``).

F.conv2d with each BatchNorm folded into its conv, F.relu, the pools, F.interpolate; in whatever dtype the state_dict and input
come in (float64 for the fixture comparisons).  Pinned to tests/golden/fid.pt on the CPU (tests/test_host_inception.py); the GPU
tests use it at sizes and batches the fixture does not hold.  Also builds the synthetic weights of the fixture from its seed."""
import os

import torch
import torch.nn.functional as F

from oracle import synth

BN_EPS = 1e-3

# (name, Cout, Cin, kh, kw): every BasicConv2d of the plan in state_dict order
A_CONVS = [("branch1x1", 64, None, 1, 1), ("branch5x5_1", 48, None, 1, 1), ("branch5x5_2", 64, 48, 5, 5),
           ("branch3x3dbl_1", 64, None, 1, 1), ("branch3x3dbl_2", 96, 64, 3, 3), ("branch3x3dbl_3", 96, 96, 3, 3),
           ("branch_pool", "pf", None, 1, 1)]
B_CONVS = [("branch3x3", 384, None, 3, 3), ("branch3x3dbl_1", 64, None, 1, 1), ("branch3x3dbl_2", 96, 64, 3, 3),
           ("branch3x3dbl_3", 96, 96, 3, 3)]
C_CONVS = [("branch1x1", 192, None, 1, 1), ("branch7x7_1", "c7", None, 1, 1), ("branch7x7_2", "c7", "c7", 1, 7),
           ("branch7x7_3", 192, "c7", 7, 1), ("branch7x7dbl_1", "c7", None, 1, 1), ("branch7x7dbl_2", "c7", "c7", 7, 1),
           ("branch7x7dbl_3", "c7", "c7", 1, 7), ("branch7x7dbl_4", "c7", "c7", 7, 1), ("branch7x7dbl_5", 192, "c7", 1, 7),
           ("branch_pool", 192, None, 1, 1)]
D_CONVS = [("branch3x3_1", 192, None, 1, 1), ("branch3x3_2", 320, 192, 3, 3), ("branch7x7x3_1", 192, None, 1, 1),
           ("branch7x7x3_2", 192, 192, 1, 7), ("branch7x7x3_3", 192, 192, 7, 1), ("branch7x7x3_4", 192, 192, 3, 3)]
E_CONVS = [("branch1x1", 320, None, 1, 1), ("branch3x3_1", 384, None, 1, 1), ("branch3x3_2a", 384, 384, 1, 3),
           ("branch3x3_2b", 384, 384, 3, 1), ("branch3x3dbl_1", 448, None, 1, 1), ("branch3x3dbl_2", 384, 448, 3, 3),
           ("branch3x3dbl_3a", 384, 384, 1, 3), ("branch3x3dbl_3b", 384, 384, 3, 1), ("branch_pool", 192, None, 1, 1)]
# (prefix, kind, Cin, parameter)
MIXED = [("blocks.2.0", "A", 192, 32), ("blocks.2.1", "A", 256, 64), ("blocks.2.2", "A", 288, 64), ("blocks.2.3", "B", 288, None),
         ("blocks.2.4", "C", 768, 128), ("blocks.2.5", "C", 768, 160), ("blocks.2.6", "C", 768, 160), ("blocks.2.7", "C", 768, 192),
         ("blocks.3.0", "D", 768, None), ("blocks.3.1", "E", 1280, None), ("blocks.3.2", "E", 2048, None)]
STEM = [("blocks.0.0", 32, 3, 3, 3), ("blocks.0.1", 32, 32, 3, 3), ("blocks.0.2", 64, 32, 3, 3), ("blocks.1.0", 80, 64, 1, 1),
        ("blocks.1.1", 192, 80, 3, 3)]


def conv_list():
    """[(name, Cout, Cin, kh, kw)] of the 94 BasicConv2d in the reference's state_dict order"""
    out = list(STEM)
    for p, kind, cin, par in MIXED:
        table = {"A": A_CONVS, "B": B_CONVS, "C": C_CONVS, "D": D_CONVS, "E": E_CONVS}[kind]
        for n, co, ci, kh, kw in table:
            sub = {"pf": par, "c7": par}
            out.append((p + "." + n, sub.get(co, co), cin if ci is None else sub.get(ci, ci), kh, kw))
    return out


def layout():
    """{key: shape} of the reference's InceptionV3(output_blocks=[3]) state_dict, in its order"""
    lay = {}
    for n, co, ci, kh, kw in conv_list():
        lay[n + ".conv.weight"] = (co, ci, kh, kw)
        for s in ("weight", "bias", "running_mean", "running_var"):
            lay[n + ".bn." + s] = (co,)
        lay[n + ".bn.num_batches_tracked"] = ()
    lay["fc.weight"] = (1008, 2048)
    lay["fc.bias"] = (1008,)
    return lay


def synth_weights(seed):
    """the fixture's weights from its seed, reference layout, float32: conv / fc weights and biases from oracle.synth (U(+-1/sqrt
    fan_in)), the BN affine 1 + 0.1 N and 0.1 N; running statistics 0 / 1 (the fixture stores the calibrated ones)"""
    lay = layout()
    wl = {k: v for k, v in lay.items() if k.endswith("conv.weight") or k.startswith("fc.")}
    sd = synth.synth_state_dict(wl, seed)
    for i, (n, co, _, _, _) in enumerate(conv_list()):
        sd[n + ".bn.weight"] = 1.0 + 0.1 * synth.randn_seeded((co,), seed * 1000 + 2 * i + 1)
        sd[n + ".bn.bias"] = 0.1 * synth.randn_seeded((co,), seed * 1000 + 2 * i + 2)
        sd[n + ".bn.running_mean"] = torch.zeros(co)
        sd[n + ".bn.running_var"] = torch.ones(co)
        sd[n + ".bn.num_batches_tracked"] = torch.tensor(0, dtype=torch.long)
    return {k: sd[k] for k in lay}


def to_torchvision_keys(sd):
    """reference InceptionV3 keys -> the pytorch-fid weight file's torchvision keys"""
    names = {"blocks.0.0": "Conv2d_1a_3x3", "blocks.0.1": "Conv2d_2a_3x3", "blocks.0.2": "Conv2d_2b_3x3", "blocks.1.0": "Conv2d_3b_1x1",
             "blocks.1.1": "Conv2d_4a_3x3", "blocks.2.0": "Mixed_5b", "blocks.2.1": "Mixed_5c", "blocks.2.2": "Mixed_5d",
             "blocks.2.3": "Mixed_6a", "blocks.2.4": "Mixed_6b", "blocks.2.5": "Mixed_6c", "blocks.2.6": "Mixed_6d",
             "blocks.2.7": "Mixed_6e", "blocks.3.0": "Mixed_7a", "blocks.3.1": "Mixed_7b", "blocks.3.2": "Mixed_7c"}
    out = {}
    for k, v in sd.items():
        p = ".".join(k.split(".")[:3])
        out[names[p] + k[len(p):] if p in names else k] = v
    return out


class Restated:
    """the network on a reference-layout state_dict; BN folded once, in float64, then cast to the state_dict's dtype"""

    def __init__(self, sd):
        self.dtype = sd["fc.weight"].dtype
        self.w, self.b = {}, {}
        for n, *_ in conv_list():
            g, bt = sd[n + ".bn.weight"].double(), sd[n + ".bn.bias"].double()
            m, v = sd[n + ".bn.running_mean"].double(), sd[n + ".bn.running_var"].double()
            s = g / torch.sqrt(v + BN_EPS)
            self.w[n] = (sd[n + ".conv.weight"].double() * s[:, None, None, None]).to(self.dtype)
            self.b[n] = (bt - m * s).to(self.dtype)
        self.fc_w, self.fc_b = sd["fc.weight"], sd["fc.bias"]

    def c(self, n, x, stride=1, padding=0):
        return F.relu(F.conv2d(x, self.w[n], self.b[n], stride=stride, padding=padding))

    @staticmethod
    def avg(x):
        return F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=False)

    def block_a(self, p, x):
        b1 = self.c(p + ".branch1x1", x)
        b5 = self.c(p + ".branch5x5_2", self.c(p + ".branch5x5_1", x), padding=2)
        b3 = self.c(p + ".branch3x3dbl_3", self.c(p + ".branch3x3dbl_2", self.c(p + ".branch3x3dbl_1", x), padding=1), padding=1)
        bp = self.c(p + ".branch_pool", self.avg(x))
        return torch.cat([b1, b5, b3, bp], 1)

    def block_b(self, p, x):
        b3 = self.c(p + ".branch3x3", x, stride=2)
        bd = self.c(p + ".branch3x3dbl_3", self.c(p + ".branch3x3dbl_2", self.c(p + ".branch3x3dbl_1", x), padding=1), stride=2)
        return torch.cat([b3, bd, F.max_pool2d(x, kernel_size=3, stride=2)], 1)

    def block_c(self, p, x):
        b1 = self.c(p + ".branch1x1", x)
        b7 = self.c(p + ".branch7x7_1", x)
        b7 = self.c(p + ".branch7x7_2", b7, padding=(0, 3))
        b7 = self.c(p + ".branch7x7_3", b7, padding=(3, 0))
        bd = self.c(p + ".branch7x7dbl_1", x)
        bd = self.c(p + ".branch7x7dbl_2", bd, padding=(3, 0))
        bd = self.c(p + ".branch7x7dbl_3", bd, padding=(0, 3))
        bd = self.c(p + ".branch7x7dbl_4", bd, padding=(3, 0))
        bd = self.c(p + ".branch7x7dbl_5", bd, padding=(0, 3))
        bp = self.c(p + ".branch_pool", self.avg(x))
        return torch.cat([b1, b7, bd, bp], 1)

    def block_d(self, p, x):
        b3 = self.c(p + ".branch3x3_2", self.c(p + ".branch3x3_1", x), stride=2)
        b7 = self.c(p + ".branch7x7x3_1", x)
        b7 = self.c(p + ".branch7x7x3_2", b7, padding=(0, 3))
        b7 = self.c(p + ".branch7x7x3_3", b7, padding=(3, 0))
        b7 = self.c(p + ".branch7x7x3_4", b7, stride=2)
        return torch.cat([b3, b7, F.max_pool2d(x, kernel_size=3, stride=2)], 1)

    def block_e(self, p, x, max_pool):
        b1 = self.c(p + ".branch1x1", x)
        b3 = self.c(p + ".branch3x3_1", x)
        b3 = torch.cat([self.c(p + ".branch3x3_2a", b3, padding=(0, 1)), self.c(p + ".branch3x3_2b", b3, padding=(1, 0))], 1)
        bd = self.c(p + ".branch3x3dbl_2", self.c(p + ".branch3x3dbl_1", x), padding=1)
        bd = torch.cat([self.c(p + ".branch3x3dbl_3a", bd, padding=(0, 1)), self.c(p + ".branch3x3dbl_3b", bd, padding=(1, 0))], 1)
        pooled = F.max_pool2d(x, kernel_size=3, stride=1, padding=1) if max_pool else self.avg(x)
        return torch.cat([b1, b3, bd, self.c(p + ".branch_pool", pooled)], 1)

    def forward(self, inp, resize_input=True, normalize_input=True):
        """inp [B, 3, H, W] in [0, 1] -> ([block 0, 1, 2 NCHW maps, block 3 [B, 2048, 1, 1]], logits [B, 1008])"""
        x = inp.to(self.dtype)
        if resize_input:
            x = F.interpolate(x, size=(299, 299), mode='bilinear', align_corners=False)
        if normalize_input:
            x = 2 * x - 1
        outs = []
        x = self.c("blocks.0.0", x, stride=2)
        x = self.c("blocks.0.1", x)
        x = self.c("blocks.0.2", x, padding=1)
        x = F.max_pool2d(x, kernel_size=3, stride=2)
        outs.append(x)
        x = self.c("blocks.1.0", x)
        x = self.c("blocks.1.1", x)
        x = F.max_pool2d(x, kernel_size=3, stride=2)
        outs.append(x)
        for p, kind, _, _ in MIXED[:8]:
            x = getattr(self, "block_" + kind.lower())(p, x)
        outs.append(x)
        x = self.block_d("blocks.3.0", x)
        x = self.block_e("blocks.3.1", x, False)
        x = self.block_e("blocks.3.2", x, True)
        x = F.adaptive_avg_pool2d(x, (1, 1))
        outs.append(x)
        logits = F.linear(torch.flatten(x, 1), self.fc_w.to(self.dtype), self.fc_b.to(self.dtype))
        return outs, logits


def fixture_state_dict(golden):
    """the fixture's full state_dict (float32): weights from its seed, running statistics as stored"""
    sd = synth_weights(golden["seed"])
    for k, v in golden["running_stats"].items():
        sd[k] = v.clone()
    return sd


def fixture_input(case):
    """the seeded [B, 3, H, W] float32 input in [0, 1) of one fixture case"""
    return torch.rand((case["B"], 3, case["H"], case["W"]), generator=torch.Generator().manual_seed(case["seed"]))


def write_weight_file(torch_home, sd):
    """sd (reference layout) saved as the pytorch-fid weight file (torchvision keys, no num_batches_tracked) where
    fid_inception_v3 looks for it under TORCH_HOME = torch_home; returns the file's path"""
    d = os.path.join(torch_home, "hub", "checkpoints")
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, "pt_inception-2015-12-05-6726825d.pth")
    tv = {k: v for k, v in to_torchvision_keys(sd).items() if not k.endswith("num_batches_tracked")}
    torch.save(tv, path)
    return path
