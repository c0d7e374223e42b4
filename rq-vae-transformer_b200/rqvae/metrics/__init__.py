"""rqvae.metrics (reference: rqvae/metrics/__init__.py:15-17).

FID runs on the native Inception engine (fid.py, inception.py) from the pytorch-fid weight file in the torch hub cache, and per-image
CLIP scores on the native CLIP engine (clip_score.clip_score).  IS needs torchvision's ImageNet Inception, and the dataset-level
CLIP score reads caption datasets, neither of which ships here: compute_IS and compute_clip_score stay placeholders that raise
NotImplementedError.  The sampling scripts import these names at module load; they only call them when
statistics are requested (`--no-stats-saving` skips them, main_sampling_fid.py:256)."""
from .fid import compute_fid, compute_rfid, compute_statistics_from_files


def _unavailable(name):
    def fn(*a, **k):
        raise NotImplementedError("rqb200: %s is out of scope (needs torchvision's ImageNet Inception or CLIP); run the "
                                  "sampling script with --no-stats-saving, or call rqvae.metrics.compute_fid (or "
                                  "rqvae.metrics.clip_score.clip_score per batch) directly" % name)
    fn.__name__ = name
    return fn


compute_IS = _unavailable("compute_IS")
compute_clip_score = _unavailable("compute_clip_score")
