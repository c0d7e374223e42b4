"""Parameter holders of rqvae/models/rqtransformer/primitives.py: ``TupleEmbedding``, ``BatchLinear`` and ``LogitMask``.

Same module path, class names, parameter / buffer names, shapes and default initialisation as the reference, so that state_dicts
load unchanged and a seeded constructor draws the reference's weights.  The arithmetic runs in the native AR engine
(RQTransformer.sample / forward); calling these modules directly raises."""
from itertools import accumulate

import torch
import torch.nn as nn


def _no_compute(self, *a, **k):
    raise RuntimeError("rqb200: parameter holder -- compute runs in the native engine (RQTransformer.sample)")


class TupleEmbedding(nn.Embedding):
    """One table per depth stacked into ``weight`` [sum(V_d), E]; code d of a tuple indexes rows ``offsets[d]`` + code.

    Initialisation: N(0, 0.02), drawn twice (once by ``nn.Embedding.__init__``, which calls ``reset_parameters``, and once more
    after the ``offsets`` buffer is registered), as the reference does."""

    def __init__(self, num_embeddings, embedding_dim, **kwargs):
        if "padding_idx" in kwargs:
            raise ValueError("padding_idx argument not supported")
        sizes = (num_embeddings,) if isinstance(num_embeddings, int) else num_embeddings
        self.num_embeddings_per_dict = sizes
        self.embedding_dim = embedding_dim
        super().__init__(num_embeddings=sum(sizes), embedding_dim=embedding_dim, **kwargs)
        starts = [0] + list(accumulate(sizes))[:-1]
        self.register_buffer("offsets", torch.tensor(starts, dtype=torch.long))
        self.reset_parameters()

    def reset_parameters(self):
        self.weight.data.normal_(mean=0.0, std=0.02)

    forward = _no_compute


class LogitMask(nn.Module):
    """Masks the logits of depth d beyond its own vocabulary V_d.  No parameters; a no-op when every depth has the same V."""

    def __init__(self, vocab_size, value=-1e6):
        super().__init__()
        self.vocab_size = vocab_size
        self.mask_cond = [vocab_size[0]] * len(vocab_size) != vocab_size
        self.value = value

    forward = _no_compute


class BatchLinear(nn.Module):
    """``n_vectors`` independent linear maps: ``weight`` [n, in, out] (input-major, the transpose of nn.Linear's), ``bias`` [n, out].
    Initialisation: weight N(0, 0.02), bias zero."""

    def __init__(self, n_vectors, in_features, out_features, bias=True):
        super().__init__()
        self.n_vectors, self.in_features, self.out_features = n_vectors, in_features, out_features
        self.weight = nn.Parameter(torch.empty(n_vectors, in_features, out_features))
        if bias:
            self.bias = nn.Parameter(torch.empty(n_vectors, out_features))
        else:
            self.register_parameter("bias", None)
        self.reset_parameters()

    def reset_parameters(self):
        self.weight.data.normal_(mean=0.0, std=0.02)
        if self.bias is not None:
            self.bias.data.zero_()

    forward = _no_compute

    def extra_repr(self):
        return "n_vectors=%d, in_features=%d, out_features=%d, bias=%s" % (self.n_vectors, self.in_features, self.out_features,
                                                                           self.bias is not None)
