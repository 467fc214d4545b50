"""The dueling head's fp32 arithmetic on the CPU (k_head_duel, csrc/net.cu; the rules are in include/b200dqn.h), so that
the device's advantages, V, Q, dZ4 and fc2's gradient compare bit for bit when they are fed the device's own H4 and
deltas, and a whole-network numpy dueling step for the trajectory bars.

Shapes (Neon layout): H4 (rows, 1024), units [0, 512) the advantage stream and [512, 1024) the value stream; W5
(A + 1, 512), rows 0..A-1 over the advantage units and row A over the value units.

Rules:
  1. A_a = head_oracle rule 1 on (H4[:, :512], W5[a]); V = the same rule on (H4[:, 512:], W5[A]).
  2. m = (sum_j A_j, j order, from 0.f) / A; Q_a = V + (A_a - m).  Every operation is one fp32 rounding.
  3. With d the row's delta at the taken action a (clipped, importance-weighted): g = d / A, dA_j = d - g at j = a and
     -g elsewhere, dV = d.  dZ4 on advantage unit k = (sum_j dA_j W5[j][k], j order, from 0.f), on value unit k =
     d W5[A][k], each +0 where H4 <= 0.
  4. fc2's per-row partials are P_b[j][k] = H4[b][k] dA_j (j < A) and P_b[A][k] = H4[b][512 + k] d, reduced over the
     rows by head_oracle's tree8 (k_optimizer / k_opt_small).
"""
import numpy as np

import head_oracle as H

F32 = np.float32
HIDDEN = 512


def streams(h4, w5):
    """Rule 1: ((rows, A) advantages, (rows,) V)."""
    h4, w5 = np.asarray(h4, F32), np.asarray(w5, F32)
    A = len(w5) - 1
    return H.q_rows(h4[:, :HIDDEN], w5[:A]), H.q_rows(h4[:, HIDDEN:], w5[A:])[:, 0]


def aggregate(adv, val, skip_mean=False, mean_div=None):
    """Rule 2: (rows, A) Q.  skip_mean / mean_div: wrong variants for showing that a test can tell them apart."""
    adv, val = np.asarray(adv, F32), np.asarray(val, F32)
    A = adv.shape[1]
    s = np.zeros(len(adv), F32)
    for j in range(A):
        s = (s + adv[:, j]).astype(F32)
    m = (s / F32(A if mean_div is None else mean_div)).astype(F32)
    if skip_mean:
        m = np.zeros_like(m)
    return (val[:, None] + (adv - m[:, None]).astype(F32)).astype(F32)


def q_rows(h4, w5):
    return aggregate(*streams(h4, w5))


def stream_grads(d, actions, A, drop_mean_term=False):
    """Rule 3's (rows, A) dA and (rows,) dV from the (rows,) deltas at the taken actions."""
    d = np.asarray(d, F32)
    g = (d / F32(A)).astype(F32)
    dA = np.repeat(-g[:, None], A, axis=1)
    rows = np.arange(len(d))
    dA[rows, actions] = d if drop_mean_term else (d - g).astype(F32)
    return dA, d.copy()


def dz4(h4, w5, dA, dV):
    """Rule 3's (rows, 1024) dZ4."""
    h4, w5 = np.asarray(h4, F32), np.asarray(w5, F32)
    A = dA.shape[1]
    adv = np.zeros((len(h4), HIDDEN), F32)
    for j in range(A):
        adv = (adv + (dA[:, j:j + 1] * w5[j][None, :]).astype(F32)).astype(F32)
    val = (dV[:, None] * w5[A][None, :]).astype(F32)
    out = np.concatenate([adv, val], axis=1)
    return np.where(h4 > 0, out, F32(0)).astype(F32)


def row_partials(h4, dA, dV):
    """Rule 4's (rows, A + 1, 512) per-row partials."""
    h4 = np.asarray(h4, F32)
    adv = (dA[:, :, None] * h4[:, None, :HIDDEN]).astype(F32)
    val = (dV[:, None, None] * h4[:, None, HIDDEN:]).astype(F32)
    return np.concatenate([adv, val], axis=1)


def fc2_grad(h4, dA, dV):
    """Rule 4: dW5 (A + 1, 512)."""
    return H.tree8(row_partials(h4, dA, dV))


# ---------------------------------------------------------------------------------------------------- whole network
def expand_w5(w5):
    """(A + 1, 512) block fc2 -> the equivalent dense (A + 1, 1024) layer over both streams."""
    A = len(w5) - 1
    full = np.zeros((A + 1, 2 * HIDDEN), F32)
    full[:A, :HIDDEN] = w5[:A]
    full[A, HIDDEN:] = w5[A]
    return full


def fold_w5(full):
    """The blocks of a dense (A + 1, 1024) fc2 gradient that the dueling fc2 has."""
    A = len(full) - 1
    return np.concatenate([full[:A, :HIDDEN], full[A:, HIDDEN:]], axis=0).astype(F32)


def forward(weights, states, keep=False):
    """oracle.dqn_oracle.forward with the dueling head: (rows, A) Q (and the activations with keep)."""
    from oracle import dqn_oracle as O
    ws = list(weights[:4]) + [expand_w5(weights[4])]
    out, acts = O.forward(ws, states, keep=True)
    A = len(weights[4]) - 1
    q = aggregate(out[:, :A], out[:, A])
    return (q, acts) if keep else q


def xavier_init(num_actions, seed):
    """Xavier draws in oracle.dqn_oracle's order for the dueling shapes: fc1 (1024, 3136), fc2 (A + 1, 512)."""
    from oracle import dqn_oracle as O
    rng = np.random.RandomState(seed)
    shapes = O.layer_shapes(num_actions)[:3] + [(2 * HIDDEN, 3136), (num_actions + 1, HIDDEN)]
    ws = []
    for i, shp in enumerate(shapes):
        s = np.sqrt(3.0 / (shp[0] if i < 3 else shp[1]))
        ws.append(rng.uniform(-s, s, shp).astype(F32))
    return ws


def numpy_step(weights, states, target_weights, minibatch, double=False, discount=0.99, lr=0.00025, decay=0.95):
    """One whole-network dueling step in numpy (oracle.dqn_oracle's backward and RMSProp through the dense form of the
    head; the one-step target, Double DQN's with double).  Updates weights / states (RMSProp planes) in place; returns
    (cost, grads)."""
    import nstep_oracle as NS
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    actions = np.asarray(actions, np.int64)
    preq, acts = forward(weights, pre, keep=True)
    postq = forward(target_weights, post)
    oq = forward(weights, post) if double else None
    deltas, row_cost, _ = NS.head_restated(preq, postq, actions, rewards, terminals, discount=discount, online_postq=oq)
    A = preq.shape[1]
    dA, dV = stream_grads(deltas[np.arange(len(actions)), actions], actions, A)
    ws = list(weights[:4]) + [expand_w5(weights[4])]
    grads = O.backward(ws, acts, np.concatenate([dA, dV[:, None]], axis=1))
    grads[4] = fold_w5(grads[4])
    O.rmsprop_update(weights, states, grads, len(actions), lr=lr, decay=decay)
    return float(np.mean(row_cost)), grads
