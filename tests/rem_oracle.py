"""The random ensemble mixture head (REM, Agarwal, Schuurmans and Norouzi, 2020) on the CPU: a numpy restatement of the
device's k_rem_alpha and k_head_rem (csrc/net.cu), with fc2 and its gradient as k_fc2_dist and k_opt_fc2_dist form them,
so that every output compares bit for bit when it is fed the device's own inputs.  A = actions, K = heads, a the taken
action, z the slot (0 online on the prestates, 1 target on the poststates, 2 online on the poststates under Double DQN).
Every operation is fp32 with its own rounding unless marked fp64 (numpy's float32 operators round once each and never
contract).

Rules (include/b200dqn.h states them too):
  1. Mixture draw: u_k = (2 m_k + 1) 2^-24, m_k from tests/iqn_oracle.py rule 1's hash at (z, b, j) = (0, 0, k) with
     rem_seed and the mixture's counter; S = sum_k double(u_k) in fp64, k order; alpha_k = float32(double(u_k) / S).
  2. theta[z][b][a * K + k] = sum_i H4[z][b][i] * W5[i][a * K + k], i = 0..511 in order: tests/c51_oracle.py rule 2.
  3. Train-step Q[z][a] = sum_k alpha_k * theta[z][b][a K + k] in k order (product rounded, then the sum).
  4. Predict Q[a] = (sum_k theta[a][k] in k order) / float32(K): tests/qr_oracle.py rule 3.
  5. The scalar head's TD step on rule 3's Q: maxq = max of slot 1's Q (slot 1's Q at the first maximum of slot 2's
     with Double DQN); y = fma(g, maxq, R) one-step, R + g * maxq n-step, R at a terminal (g = 0); target = float32(y);
     delta = Q[0][a] - target; row cost 0.5 * delta * delta (times w on a prioritized ring, whose TD error is delta);
     d = clip(delta) (no clip at clip_error 0), times w on a prioritized ring.
  6. dtheta[a][k] = alpha_k * d at the taken action, 0 elsewhere.
  7. dZ4, its fp16 planes, the dW5 row partials and fc2's gradient: tests/c51_oracle.py rules 10 and 11 with gl = dtheta.
"""
import numpy as np

import c51_oracle as C51
import iqn_oracle as IQ
import qr_oracle as QR
from munchausen_oracle import fma

F32 = np.float32

logits = C51.logits             # rule 2
first_argmax = C51.first_argmax
one_step_return = C51.one_step_return
n_step_return = C51.n_step_return
predict_q = QR.q_values         # rule 4
dz4 = C51.dz4                   # rule 7
fp16_planes = C51.fp16_planes
fc2_grad = C51.fc2_grad


def draws(seed, ctr, k):
    """Rule 1's u: (K,) float32, every value an exact (2m + 1) 2^-24."""
    return IQ.tau_draw(seed, ctr, 1, 1, k)[0]


def alpha(seed, ctr, k):
    """Rule 1: (K,) float32 mixture of the draw at counter value ctr."""
    u = [float(v) for v in draws(seed, ctr, k)]
    s = 0.0
    for v in u:
        s += v
    return np.array([F32(v / s) for v in u], F32)


def mixed_q(theta, al):
    """Rule 3 on the last axis of theta (.., K)."""
    theta, al = np.asarray(theta, F32), np.asarray(al, F32)
    q = np.zeros(theta.shape[:-1], F32)
    for k in range(theta.shape[-1]):
        q = q + al[k] * theta[..., k]
    return q


def td_step(qpre, qpost, qonline_post, a, R, g, clip, nstep=False, w=None):
    """Rule 5 for one sample on rule 3's fp32 rows: (target, delta, row cost, d)."""
    qpost = np.asarray(qpost, F32)
    maxq = float(qpost[first_argmax(qonline_post)] if qonline_post is not None else qpost.max())
    if g == 0:
        y = float(R)
    else:
        y = float(R) + float(g) * maxq if nstep else fma(float(g), maxq, float(R))
    target = F32(y)
    delta = F32(F32(qpre[a]) - target)
    cost = F32(F32(F32(0.5) * delta) * delta)
    d = delta
    if w is not None:
        cost = F32(F32(w) * cost)
    if clip:
        d = F32(min(max(d, -F32(clip)), F32(clip)))
    if w is not None:
        d = F32(d * F32(w))
    return target, delta, cost, d


def head(theta, al, actions, returns, clip, double=False, nstep=False, w=None):
    """Rules 3, 5 and 6 on the device's (3, batch, A, K) theta: (Q of the three slots, targets, deltas, row costs,
    dtheta (batch, K))."""
    theta = np.asarray(theta, F32)
    q = mixed_q(theta, al)
    n, K = len(actions), theta.shape[-1]
    T, D, cost, g = np.zeros(n, F32), np.zeros(n, F32), np.zeros(n, F32), np.zeros((n, K), F32)
    for b in range(n):
        R, gam = returns[b]
        T[b], D[b], cost[b], d = td_step(q[0, b], q[1, b], q[2, b] if double else None, int(actions[b]), R, gam, clip,
                                         nstep, None if w is None else w[b])
        g[b] = (np.asarray(al, F32) * d).astype(F32)
    return q, T, D, cost, g


def numpy_step(weights, states, target_weights, minibatch, nh, al, clip=1.0, discount=0.99, min_reward=-1,
               max_reward=1, lr=0.00025, decay=0.95):
    """One whole-network REM step in numpy at mixture al (oracle.dqn_oracle's forward, backward and RMSProp with this
    head): the trajectory yardstick.  Updates weights / states (RMSProp planes) in place; returns (cost, grads, dtheta)."""
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    th_pre, acts = O.forward(weights, pre, keep=True)              # (B, A*K): H4 @ W5^T
    th_post = O.forward(target_weights, post)
    B = len(actions)
    A = th_pre.shape[1] // nh
    q_pre, q_post = mixed_q(th_pre.reshape(B, A, nh), al), mixed_q(th_post.reshape(B, A, nh), al)
    deltas = np.zeros((B, A * nh), F32)
    g = np.zeros((B, nh), F32)
    cost = 0.0
    for b in range(B):
        a = int(actions[b])
        R, gam = one_step_return(rewards[b], terminals[b], discount, min_reward, max_reward)
        _, _, c, d = td_step(q_pre[b], q_post[b], None, a, R, gam, clip)
        g[b] = (np.asarray(al, F32) * d).astype(F32)
        deltas[b, a * nh:(a + 1) * nh] = g[b]
        cost += float(c)
    grads = O.backward(weights, acts, deltas)
    O.rmsprop_update(weights, states, grads, B, lr=lr, decay=decay)
    return cost / B, grads, g
