"""Bootstrapped DQN heads (Osband, Blundell, Pritzel and Van Roy, 2016) on the CPU: a numpy restatement of the device's
k_head_boot and k_boot_predict (csrc/net.cu), with fc2 and its gradient as k_fc2_dist and k_opt_fc2_dist form them, so
that every output compares bit for bit when it is fed the device's own inputs.  A = actions, K = heads, b the sample, a
the taken action, z the slot (0 online on the prestates, 1 target on the poststates, 2 online on the poststates under
Double DQN), i the ring slot of the sample's transition.  Every operation is fp32 with its own rounding unless marked
fp64 (numpy's float32 operators round once each and never contract).

Rules (include/b200dqn.h states them too):
  1. Masks: m_k = [double(u) < p], u = tests/rem_oracle.py rule 1's draw (2m + 1) 2^-24 at counter value i, head k,
     with bootstrap_seed.  At p = 1 every mask is 1.
  2. theta[z][b][a * K + k] = sum_i H4[z][b][i] * W5[i][a * K + k]: tests/rem_oracle.py rule 2.
  3. a*_k = the first maximum over a of slot 1's theta[.][a][k] (slot 2's with Double DQN); y_k = fma(g, q', R) one-step,
     R + g * q' n-step, R at a terminal (g = 0), q' = slot 1's theta at (a*_k, k); target_k = float32(y_k);
     delta_k = theta[0][b][a][k] - target_k.
  4. Row cost = (sum over unmasked k of 0.5 * delta_k * delta_k, k order) / K, times w on a prioritized ring; TD error
     (sum_k |delta_k| in k order) / K over every head; d_k = clip(delta_k) (no clip at clip_error 0), times w on a
     prioritized ring; dtheta_k = m_k ? d_k : 0 at the taken action, 0 elsewhere.
  5. dZ4 = H4 > 0 ? (sum_k W5[t][a K + k] * dtheta_k in k order) / K : 0 with the fp16 planes every head writes; fc2's
     gradient is tests/c51_oracle.py rule 11 with the full dtheta.
  6. The Q rows of a train step: rule 7 at h = -1.
  7. Predict at the active head h: h = -1 the mean over the heads (tests/qr_oracle.py rule 3), h >= 0 theta[a][h].
"""
import numpy as np

import c51_oracle as C51
import rem_oracle as REM
from munchausen_oracle import fma

F32 = np.float32

logits = C51.logits                     # rule 2
first_argmax = C51.first_argmax
one_step_return = C51.one_step_return
n_step_return = C51.n_step_return
fp16_planes = C51.fp16_planes
fc2_grad = C51.fc2_grad                 # rule 5, with the full dtheta


def uniforms(seed, slot, K):
    """Rule 1's u of ring slot `slot`: (K,) float32, every value an exact (2m + 1) 2^-24."""
    return REM.draws(seed, slot, K)


def masks(seed, slots, K, p):
    """Rule 1: (len(slots), K) uint8 masks of the given ring slots."""
    return np.array([[1 if float(u) < float(p) else 0 for u in uniforms(seed, int(i), K)] for i in slots], np.uint8)


def predict_q(theta, h=-1):
    """Rule 7 on the last axis of theta (.., K)."""
    theta = np.asarray(theta, F32)
    if h >= 0:
        return theta[..., h].copy()
    return REM.predict_q(theta)


def td_step(th_pre, th_post, th_choice, a, R, g, m, clip, nstep=False, w=None):
    """Rules 3 and 4 for one sample on its (A, K) theta rows: (targets, deltas, row cost, TD error, dtheta (K,))."""
    th_pre, th_post, th_choice = (np.asarray(x, F32) for x in (th_pre, th_post, th_choice))
    K = th_pre.shape[1]
    T, D, G = np.zeros(K, F32), np.zeros(K, F32), np.zeros(K, F32)
    cost, err = F32(0), F32(0)
    for k in range(K):
        qn = float(th_post[first_argmax(th_choice[:, k]), k])
        if g == 0:
            y = float(R)
        else:
            y = float(R) + float(g) * qn if nstep else fma(float(g), qn, float(R))
        T[k] = F32(y)
        D[k] = F32(th_pre[a, k] - T[k])
        d = D[k]
        if clip:
            d = F32(min(max(d, -F32(clip)), F32(clip)))
        if w is not None:
            d = F32(d * F32(w))
        G[k] = d if m[k] else F32(0)
        if m[k]:
            cost = F32(cost + F32(F32(F32(0.5) * D[k]) * D[k]))
        err = F32(err + abs(D[k]))
    cost, err = F32(cost / F32(K)), F32(err / F32(K))
    if w is not None:
        cost = F32(F32(w) * cost)
    return T, D, cost, err, G


def head(theta, actions, returns, m, clip, double=False, nstep=False, w=None):
    """Rules 3, 4 and 6 on the device's (3, batch, A, K) theta and (batch, K) masks: (Q of the three slots, targets,
    deltas, row costs, TD errors, dtheta (batch, K))."""
    theta = np.asarray(theta, F32)
    q = predict_q(theta)
    n, K = len(actions), theta.shape[-1]
    T, D, G = np.zeros((n, K), F32), np.zeros((n, K), F32), np.zeros((n, K), F32)
    cost, err = np.zeros(n, F32), np.zeros(n, F32)
    for b in range(n):
        R, gam = returns[b]
        T[b], D[b], cost[b], err[b], G[b] = td_step(theta[0, b], theta[1, b], theta[2 if double else 1, b],
                                                    int(actions[b]), R, gam, m[b], clip, nstep,
                                                    None if w is None else w[b])
    return q, T, D, cost, err, G


def dz4(h4_row, w5_internal, a, g):
    """Rule 5 for one sample: the mean over the heads of the heads' gradients into H4."""
    K = len(g)
    blk = np.asarray(w5_internal, F32)[:, a * K:(a + 1) * K]
    acc = np.zeros(blk.shape[0], F32)
    for k in range(K):
        acc = acc + blk[:, k] * F32(g[k])
    return np.where(np.asarray(h4_row) > 0, (acc / F32(K)).astype(F32), F32(0)).astype(F32)


def numpy_step(weights, states, target_weights, minibatch, K, m, clip=1.0, discount=0.99, min_reward=-1,
               max_reward=1, lr=0.00025, decay=0.95):
    """One whole-network bootstrapped step in numpy with masks m (batch, K) (oracle.dqn_oracle's forward, backward and
    RMSProp with this head): the trajectory yardstick.  Updates weights / states (RMSProp planes) in place; returns
    (cost, grads, dtheta)."""
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    th_pre, acts = O.forward(weights, pre, keep=True)              # (B, A*K): H4 @ W5^T
    th_post = O.forward(target_weights, post)
    B = len(actions)
    A = th_pre.shape[1] // K
    th_pre, th_post = th_pre.reshape(B, A, K), th_post.reshape(B, A, K)
    deltas = np.zeros((B, A * K), F32)
    g = np.zeros((B, K), F32)
    cost = 0.0
    for b in range(B):
        a = int(actions[b])
        R, gam = one_step_return(rewards[b], terminals[b], discount, min_reward, max_reward)
        _, _, c, _, g[b] = td_step(th_pre[b], th_post[b], th_post[b], a, R, gam, m[b], clip)
        deltas[b, a * K:(a + 1) * K] = g[b]
        cost += float(c)
    grads = O.backward(weights, acts, (deltas / F32(K)).astype(F32))   # the shared network sees the mean
    grads[4] = (deltas.T @ acts["h4"]).astype(F32)                      # the heads their full dtheta
    O.rmsprop_update(weights, states, grads, B, lr=lr, decay=decay)
    return cost / B, grads, g
