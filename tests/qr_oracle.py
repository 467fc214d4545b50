"""The quantile-regression value head (QR-DQN, Dabney, Rowland, Bellemare and Munos, 2018) on the CPU: a numpy
restatement of the device's k_fc2_dist, k_head_qr and k_opt_fc2_dist (csrc/net.cu), so that every output compares bit
for bit when it is fed the device's own inputs.  A = actions, N = quantiles, a the taken action, z the slot (0 online on
the prestates, 1 target on the poststates, 2 online on the poststates under Double DQN).  Every operation is fp32 with
its own rounding unless marked fp64 (numpy's float32 operators round once each and never contract).

Rules (include/b200dqn.h states them too):
  1. Midpoints (fp64): tau_i = (2i + 1) / 2N; wlo_i = float32(tau_i) weighs u >= 0, whi_i = float32((2N - 2i - 1) / 2N)
     weighs u < 0.
  2. theta[z][b][a * N + i] = sum_k H4[z][b][k] * W5[k][a * N + i], k = 0..511 in order: tests/c51_oracle.py rule 2.
  3. Q[a] = (sum_i theta[a][i] in i order) / float32(N).
  4. a* = first index of the maximum of slot 1's Q (slot 2's with Double DQN); q'_j = theta[1][b][a* N + j].
  5. Return (fp64): R and g as tests/c51_oracle.py rule 6 (g = 0 when the window holds a terminal);
     T_j = float32(R + g * double(q'_j)).
  6. u_ij = T_j - theta[0][b][a N + i].
  7. w_ij = whi_i if u_ij < 0 else wlo_i.
  8. kappa > 0: L = 0.5 * (u * u) if |u| <= kappa else kappa * (|u| - 0.5 * kappa); rho_ij = (w * L) / kappa;
     c_ij = (w * clamp(u, -kappa, kappa)) / kappa.  kappa = 0: rho_ij = w * |u|; c_ij = w if u > 0, -w if u < 0, else 0.
  9. Loss_i = (sum_j rho_ij in j order) / N; the row loss l = sum_i Loss_i in i order.  Row cost l, or isw * l on a
     prioritized ring (whose td_err is the unweighted l).
 10. dtheta_i = -((sum_j c_ij in j order) / N), times isw on a prioritized ring; 0 for every other action.
 11. dZ4, its fp16 planes and the dW5 row partials: tests/c51_oracle.py rule 10 with gl = dtheta.
 12. fc2's gradient: tests/c51_oracle.py rule 11 with gl = dtheta; then the configured optimizer.
"""
import numpy as np

import c51_oracle as C51

F32 = np.float32

logits = C51.logits             # rule 2: the same fp32 dot products as the distributional head
first_argmax = C51.first_argmax
one_step_return = C51.one_step_return
n_step_return = C51.n_step_return
dz4 = C51.dz4                   # rule 11
fp16_planes = C51.fp16_planes
fc2_grad = C51.fc2_grad         # rule 12


def taus(n):
    """Rule 1: (wlo, whi) float32."""
    wlo = np.array([(2 * i + 1) / (2 * n) for i in range(n)], np.float64).astype(F32)
    whi = np.array([(2 * n - 2 * i - 1) / (2 * n) for i in range(n)], np.float64).astype(F32)
    return wlo, whi


def q_values(theta):
    """Rule 3 on the last axis."""
    theta = np.asarray(theta, F32)
    s = np.zeros(theta.shape[:-1], F32)
    for i in range(theta.shape[-1]):
        s = s + theta[..., i]
    return s / F32(theta.shape[-1])


def targets(R, g, qprime):
    """Rule 5: T (float32) of one sample from the fp64 return and the target quantiles q'."""
    return np.array([F32(float(R) + float(g) * float(q)) for q in np.asarray(qprime, F32)], F32)


def pair_terms(T, th, kappa):
    """Rules 6-8: (rho, c), each (N_i, N_j) float32, for the taken action's quantiles th and the targets T."""
    T, th, kap = np.asarray(T, F32), np.asarray(th, F32), F32(kappa)
    wlo, whi = taus(len(th))
    u = T[None, :] - th[:, None]
    w = np.where(u < 0, whi[:, None], wlo[:, None]).astype(F32)
    au = np.abs(u)
    if kap > 0:
        L = np.where(au <= kap, F32(0.5) * (u * u), kap * (au - F32(0.5) * kap)).astype(F32)
        rho = (w * L) / kap
        c = (w * np.minimum(np.maximum(u, -kap), kap)) / kap
    else:
        rho = w * au
        c = np.where(u > 0, w, np.where(u < 0, -w, F32(0))).astype(F32)
    return rho.astype(F32), c.astype(F32)


def loss_and_grad(T, th, kappa, w=None):
    """Rules 9 and 10 for one sample: (row loss l before the importance weight, dtheta)."""
    rho, c = pair_terms(T, th, kappa)
    n = len(th)
    srho = np.zeros(n, F32)
    sc = np.zeros(n, F32)
    for j in range(n):
        srho = srho + rho[:, j]
        sc = sc + c[:, j]
    loss_i = srho / F32(n)
    l = F32(0)
    for v in loss_i:
        l = F32(l + v)
    g = -(sc / F32(n))
    if w is not None:
        g = (g * F32(w)).astype(F32)
    return l, g.astype(F32)


def head(theta, actions, returns, kappa, double=False, w=None):
    """Rules 4-10 on the device's (3, batch, A, N) theta and per-sample (R, g): (a*, T, row loss l, dtheta)."""
    theta = np.asarray(theta, F32)
    n, N = len(actions), theta.shape[-1]
    astar = np.zeros(n, np.int64)
    T = np.zeros((n, N), F32)
    loss = np.zeros(n, F32)
    g = np.zeros((n, N), F32)
    for b in range(n):
        astar[b] = first_argmax(q_values(theta[2 if double else 1, b]))
        R, gam = returns[b]
        T[b] = targets(R, gam, theta[1, b, astar[b]])
        loss[b], g[b] = loss_and_grad(T[b], theta[0, b, actions[b]], kappa, None if w is None else w[b])
    return astar, T, loss, g


def numpy_step(weights, states, target_weights, minibatch, nq, kappa=1.0, discount=0.99, min_reward=-1, max_reward=1,
               lr=0.00025, decay=0.95):
    """One whole-network QR step in numpy (oracle.dqn_oracle's forward, backward and RMSProp with this head): the
    trajectory yardstick.  Updates weights / states (RMSProp planes) in place; returns (cost, grads, T, dtheta)."""
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    th_pre, acts = O.forward(weights, pre, keep=True)              # (B, A*N): H4 @ W5^T
    th_post = O.forward(target_weights, post)
    B = len(actions)
    A = th_pre.shape[1] // nq
    th_pre, th_post = th_pre.reshape(B, A, nq), th_post.reshape(B, A, nq)
    deltas = np.zeros((B, A * nq), F32)
    T = np.zeros((B, nq), F32)
    g = np.zeros((B, nq), F32)
    cost = 0.0
    for b in range(B):
        a = int(actions[b])
        astar = first_argmax(q_values(th_post[b]))
        R, gam = one_step_return(rewards[b], terminals[b], discount, min_reward, max_reward)
        T[b] = targets(R, gam, th_post[b, astar])
        l, g[b] = loss_and_grad(T[b], th_pre[b, a], kappa)
        deltas[b, a * nq:(a + 1) * nq] = g[b]
        cost += float(l)
    grads = O.backward(weights, acts, deltas)
    O.rmsprop_update(weights, states, grads, B, lr=lr, decay=decay)
    return cost / B, grads, T, g
