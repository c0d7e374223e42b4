"""Classifier rejection sampling of a class-conditional RQ-Transformer: best-of-N by an ImageNet classifier's class log-probability.

The RQ-Transformer paper's bracketed ImageNet FIDs use "5% rejection sampling via pretrained ResNet-101"; neither the paper nor the
reference code spells out the rule.  This package's rule: every requested label gets ``candidates`` samples and keeps the one whose
``classifier.class_log_prob(pixels, label)`` is largest (ties keep the earlier candidate), so the acceptance rate is 1 / candidates and
the paper's 5 % is ``candidates=20``."""
import torch

__all__ = ["rejection_sample"]


def _check(ar, labels, candidates, batch_size):
    if isinstance(candidates, bool) or not isinstance(candidates, int) or candidates < 1:
        raise ValueError("rejection_sample: candidates must be an int >= 1, got %r" % (candidates,))
    if batch_size is not None and (isinstance(batch_size, bool) or not isinstance(batch_size, int) or batch_size < 1):
        raise ValueError("rejection_sample: batch_size must be None or an int >= 1, got %r" % (batch_size,))
    if getattr(ar, "block_size_cond", 0) != 1 or getattr(ar, "vocab_size_cond", 1) <= 1:
        raise ValueError("rejection_sample: the model has no class condition (vocab_size_cond = %s, cond_len = %s)"
                         % (getattr(ar, "vocab_size_cond", None), getattr(ar, "block_size_cond", None)))
    if not isinstance(labels, torch.Tensor) or labels.dtype.is_floating_point or labels.dtype.is_complex or labels.dtype == torch.bool \
            or labels.dim() != 1 or labels.numel() < 1:
        raise ValueError("rejection_sample: labels must be a non-empty integer [B] tensor, got %s %s"
                         % (getattr(labels, "dtype", type(labels).__name__), tuple(getattr(labels, "shape", ()))))
    if int(labels.min()) < 0 or int(labels.max()) >= ar.vocab_size_cond:
        raise ValueError("rejection_sample: labels must lie in [0, %d)" % ar.vocab_size_cond)


@torch.no_grad()
def rejection_sample(ar, vae, classifier, labels, candidates=20, batch_size=None, center_crop=224, **sample_kwargs):
    """Best-of-``candidates`` class-conditional samples.

    ar: a class-conditional RQTransformer (cond_len 1); vae: the RQ-VAE whose codes it samples (``model_aux`` and ``decode_code``);
    classifier: a module with ``class_log_prob(pixels, labels, center_crop)``, e.g. rqvae.metrics.resnet.ResNet101; labels: integer [B]
    class indices (ImageNet's sorted-wnid order, which the reference's ImageNet loader and torchvision's ResNet share).

    Round c = 0 .. candidates - 1 runs ``ar.sample(zeros, model_aux=vae, cond=labels[chunk], **sample_kwargs)`` over chunks of
    ``batch_size`` labels (default: all of them), decodes the codes with ``vae.decode_code``, maps them to [0, 1] with
    clamp(x * 0.5 + 0.5, 0, 1) (the reference's main_sampling_fid.py) and scores each image's requested label with
    ``classifier.class_log_prob(pixels, label, center_crop)``.  A candidate replaces the kept one when its score is strictly larger,
    so ties keep the earlier candidate.  Only the running best codes, pixels and scores are kept.  ``sample_kwargs`` (temperature, top_k,
    top_p, cfg_scale / uncond, amp, ...) pass straight to ``sample``; a per-image ``uncond`` is chunked with the labels.

    Returns (codes [B, H, W, D] int64, pixels [B, 3, H', W'] in [0, 1], scores [B] fp32), on the model's device."""
    _check(ar, labels, candidates, batch_size)
    dev = next(ar.parameters()).device
    labels = labels.to(device=dev, dtype=torch.int64)
    B = labels.shape[0]
    bs = batch_size or B
    uncond = sample_kwargs.pop("uncond", None)
    H, W, D = ar.block_size
    codes = pixels = scores = None
    for c in range(candidates):
        for s in range(0, B, bs):
            e = min(B, s + bs)
            kw = dict(sample_kwargs)
            if uncond is not None:
                kw["uncond"] = uncond.reshape(B, -1)[s:e]
            cand = ar.sample(torch.zeros(e - s, H, W, D, dtype=torch.long, device=dev), model_aux=vae, cond=labels[s:e, None], **kw)
            pix = torch.clamp(vae.decode_code(cand) * 0.5 + 0.5, 0, 1)
            sc = classifier.class_log_prob(pix, labels[s:e], center_crop=center_crop)
            if codes is None:
                codes = torch.empty(B, *cand.shape[1:], dtype=cand.dtype, device=dev)
                pixels = torch.empty(B, *pix.shape[1:], dtype=pix.dtype, device=dev)
                scores = torch.full((B,), float("-inf"), dtype=torch.float32, device=dev)
            better = sc.float() > scores[s:e] if c > 0 else torch.ones_like(sc, dtype=torch.bool)
            codes[s:e] = torch.where(better[:, None, None, None], cand, codes[s:e])
            pixels[s:e] = torch.where(better[:, None, None, None], pix, pixels[s:e])
            scores[s:e] = torch.where(better, sc.float(), scores[s:e])
    return codes, pixels, scores
