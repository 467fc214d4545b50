"""Restatement of global gradient-norm clipping (include/b200dqn.h, b200dqn_net_config::max_grad_norm).

With M = max_grad_norm > 0, every train step:
  1. forms gg = fl32(g / bsz) for every parameter of layers 0-4 and of the IQN / FQF embedding (layer 5): g is the
     summed gradient (get_grads()), bsz the optimizer's batch size;
  2. S_l = sum of double(gg)^2 over layer l in fp64 (exact products; here math.fsum, the exactly rounded sum);
  3. N = sqrt(S_0 + ... + S_5) in fp64, summed in layer order (S_5 = 0 without an embedding);
  4. c = M / (N + 1e-6) in fp64, c32 = float32(c) if c < 1 else 1 (a NaN N gives 1);
  5. gg' = fl32(gg c32), from which the configured optimizer continues as usual (call it with gg' and batch size 1).
The FQF fraction layer (layer 6) is neither counted nor scaled.
"""
import math

import numpy as np

F32 = np.float32


def scaled_grads(grads, bsz):
    """gg = fl32(g / bsz) of every layer."""
    return [(np.asarray(g, F32) / F32(bsz)).astype(F32) for g in grads]


def layer_sq(gg):
    """S_l of one layer, exactly rounded."""
    return math.fsum((np.asarray(gg, F32).astype(np.float64).ravel()) ** 2)


def norm_from_sq(sq):
    """N from the six S_l, summed in layer order."""
    s = 0.0
    for v in sq:
        s = s + float(v)
    return math.sqrt(s)


def clip_scale(norm, max_norm):
    """c32 of rule 4."""
    c = float(max_norm) / (float(norm) + 1e-6)
    return F32(c) if c < 1.0 else F32(1.0)


def clip(grads, bsz, max_norm):
    """(gg', S, N, c32) for the layers 0-4 (+ the embedding) in `grads`."""
    gg = scaled_grads(grads, bsz)
    sq = [layer_sq(x) for x in gg] + [0.0] * (6 - len(gg))
    n = norm_from_sq(sq)
    c = clip_scale(n, max_norm)
    return [(x * c).astype(F32) for x in gg], sq, n, c
