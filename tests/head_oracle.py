"""The scalar value head's fp32 arithmetic on the CPU: a numpy restatement of fc2's forward in k_head and of fc2's
gradient as k_optimizer and k_opt_small reduce it (csrc/net.cu), so that the device's Q rows and get_grads()[4] compare
bit for bit when they are fed the device's own H4 and deltas.  A = actions, W5 in Neon layout (A, 512), i.e. the
device's internal [512][A] transposed.

Rules:
  1. Q rows (k_head, every slot): Q[b][a] = sum over the 16 warps w of s_w, added in warp order onto 0.f, where s_w is
     lane 0 of the xor butterfly (offsets 16, 8, 4, 2, 1) over the 32 fp32 products p_k = fl(H4[b][k] * W5[a][k]),
     k = 32 w + lane.  Every product and every sum is rounded once.  The sm_90a SASS of all four k_head instantiations
     shows FMUL, then SHFL.BFLY 0x10, then FADD of the product and the shuffled value: ptxas does not contract the
     product into the first butterfly add (no FFMA there), so the products are rounded before any sum.
  2. fc2's gradient: per-row partials P_b[a][k] = fl(H4[b][k] * d_b) at the row's taken action a = act[b] and 0.f at
     every other action, with d_b the device's clipped delta (already importance-weighted on a prioritized ring).
     They are reduced over the rows by eight strided running sums s_u = sum of P_b over b = u (mod 8), b ascending,
     from 0.f, combined as ((s0 + s1) + (s2 + s3)) + ((s4 + s5) + (s6 + s7)).  k_optimizer (the serial schedule, the
     SIMT engine's fc1 + fc2 update and get_grads) writes this tree out; k_opt_small (the tensor-core branch schedule)
     gives lane l of eight the running sum s_l and combines the lanes by the xor butterfly 1, 2, 4, which is the same
     tree because an fp32 sum does not depend on the order of its two operands.
"""
import numpy as np

F32 = np.float32
HIDDEN = 512


def butterfly(x):
    """Lane 0 of the warp's xor butterfly 16, 8, 4, 2, 1 over the last axis (32 lanes), in fp32."""
    x = np.asarray(x, F32)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        x = (x + x[..., lanes ^ o]).astype(F32)
    return x[..., 0]


def q_rows(h4, w5, warp_order=None):
    """Rule 1: (rows, A) Q of a (rows, 512) H4 and a Neon (A, 512) W5.  warp_order: the order the 16 warp sums are
    added in (the device's is 0..15; others are for showing that the order is observable)."""
    h4, w5 = np.asarray(h4, F32), np.asarray(w5, F32)
    prod = (h4[:, None, :] * w5[None, :, :]).astype(F32)                 # (rows, A, 512), one rounding each
    warp = butterfly(prod.reshape(len(h4), len(w5), HIDDEN // 32, 32))  # (rows, A, 16)
    q = np.zeros((len(h4), len(w5)), F32)
    for w in (range(HIDDEN // 32) if warp_order is None else warp_order):
        q = (q + warp[:, :, w]).astype(F32)
    return q


def row_partials(h4, d, actions, num_actions):
    """Rule 2's per-row partials: (rows, A, 512)."""
    h4 = np.asarray(h4, F32)
    d = np.asarray(d, F32)
    actions = np.asarray(actions, np.int64)
    out = np.zeros((len(h4), num_actions, HIDDEN), F32)
    out[np.arange(len(h4)), actions] = (h4 * d[:, None]).astype(F32)
    return out


def tree8(parts):
    """Rule 2's reduction over the first axis."""
    s = [np.zeros(parts.shape[1:], F32) for _ in range(8)]
    for b in range(len(parts)):
        s[b % 8] = (s[b % 8] + parts[b]).astype(F32)
    return (((s[0] + s[1]) + (s[2] + s[3])) + ((s[4] + s[5]) + (s[6] + s[7]))).astype(F32)


def fc2_grad(h4, d, actions, num_actions):
    """Rule 2: dW5 in Neon layout (A, 512) from the (rows, 512) H4, the per-row clipped delta at the taken action
    (rows,) and the taken actions."""
    return tree8(row_partials(h4, d, actions, num_actions))


def sequential(parts):
    """One running sum over the rows in row order (not the device's order; for showing that the order is observable)."""
    acc = np.zeros(parts.shape[1:], F32)
    for p in parts:
        acc = (acc + p).astype(F32)
    return acc
