"""The implicit quantile network head (IQN, Dabney, Ostrovski, Silver and Munos, 2018) on the CPU: a numpy restatement of
the device's k_iqn_tau, k_iqn_phi, k_iqn_mod, k_head_iqn, k_iqn_mod_bwd and k_iqn_we (csrc/net.cu), so that every
output compares bit for bit when it is fed the device's own inputs.  N = num_tau_samples, K = num_quantile_samples, b
the sample, a the taken action, z the slot (0 online on the prestates, 1 target on the poststates).  Every operation is
fp32 with its own rounding unless marked fp64 (numpy's float32 operators round once each and never contract).

Rules (include/b200dqn.h states them too):
  1. tau = (2m + 1) 2^-24, m = the top 23 bits of the high 32 bits of
     mix(mix(seed + 0x9E3779B97F4A7C15 (ctr + 1)) ^ (z << 32 | b << 8 | j)), mix = splitmix64's finaliser, mod 2^64.
  2. Rows r = b N + j (train), r = b K + k (predict, slot 0).
  3. c[r][i] = float32(cos((pi i) tau_r)) in fp64, i = 0..63 (the device's cos: within one fp32 ulp, not bit for bit).
  4. phi[r][col] = max(0, sum_i c[r][i] We[i][col], i order).
  5. X[r] = psi[b] * phi[r], psi = H3.
  6. theta = H4 W5 (tests/c51_oracle.py rule 2 with A columns).
  7. Q[a] = (sum_j theta[b N + j][a], j order) / N.
  8. a* = first maximum of slot 1's Q.
  9. T_j = float32(R + g double(theta[1][b N + j][a*])); u_ij = T_j - theta[0][b N + i][a]; weight tau_i (u >= 0) or
     1 - tau_i (u < 0); the loss, the row cost and dtheta follow tests/qr_oracle.py rules 8-10.
 10. dZ4[r][k] = H4 > 0 ? W5[k][a] dtheta_r : 0; fc2's gradient column a = sum_r H4[r][k] dtheta_r in row order.
 12. dpsi[b][col] = (sum_j dX[r][col] phi[r][col], j order) under psi > 0; dphi = phi > 0 ? dX psi : 0.
 13. dWe[i][col] = sum_r c[r][i] dphi[r][col], row order.
"""
import numpy as np

import c51_oracle as C51
import qr_oracle as QR

F32 = np.float32
M64 = (1 << 64) - 1
FLAT = 3136

first_argmax = C51.first_argmax
one_step_return = C51.one_step_return
n_step_return = C51.n_step_return
logits = C51.logits


def _mix(x):
    x = int(x) & M64
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    x ^= x >> 31
    return x


def tau_draw(seed, ctr, nets, rows, per):
    """Rule 1: (nets, rows * per) float32 tau of the draw at counter value ctr."""
    base = _mix((int(seed) + 0x9E3779B97F4A7C15 * (int(ctr) + 1)) & M64)
    out = np.zeros((nets, rows * per), F32)
    for z in range(nets):
        for b in range(rows):
            for j in range(per):
                m = (_mix(base ^ (z << 32 | b << 8 | j)) >> 32) >> 9
                out[z, b * per + j] = F32((2 * m + 1) * 2.0 ** -24)
    return out


def cos_features(tau):
    """Rule 3 with numpy's float64 cos: (..., 64) float32."""
    i = np.arange(64, dtype=np.float64)
    return np.cos((np.pi * i) * np.asarray(tau, np.float64)[..., None]).astype(F32)


def phi(c, we):
    """Rule 4 for (rows, 64) c and a (64, cols) We in any column order."""
    c, we = np.asarray(c, F32), np.asarray(we, F32)
    acc = np.zeros((c.shape[0], we.shape[1]), F32)
    for i in range(c.shape[1]):
        acc = acc + c[:, i:i + 1] * we[i:i + 1, :]
    return np.maximum(acc, F32(0))


def modulate(psi, ph, per):
    """Rule 5: X (rows * per, cols) from psi (rows, cols) and phi."""
    return (np.repeat(np.asarray(psi, F32), per, axis=0) * np.asarray(ph, F32)).astype(F32)


def q_values(theta_rows, per):
    """Rule 7: (rows, A) Q from (rows * per, A) theta."""
    th = np.asarray(theta_rows, F32)
    th = th.reshape(th.shape[0] // per, per, th.shape[1])
    s = np.zeros((th.shape[0], th.shape[2]), F32)
    for j in range(per):
        s = s + th[:, j]
    return s / F32(per)


def pair_terms(T, th, tau, kappa):
    """Rule 9 (tests/qr_oracle.py rules 6-8 with the sampled weights): (rho, c), each (N_i, N_j) float32."""
    T, th, kap = np.asarray(T, F32), np.asarray(th, F32), F32(kappa)
    wlo = np.asarray(tau, F32)
    whi = (F32(1) - wlo).astype(F32)
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


def loss_and_grad(T, th, tau, kappa, w=None):
    """tests/qr_oracle.py rules 9 and 10 over the sampled pairs: (row loss before the importance weight, dtheta)."""
    rho, c = pair_terms(T, th, tau, kappa)
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


def head(theta, tau0, actions, returns, kappa, per, w=None):
    """Rules 7-9 on the device's (2, >= B N, A) theta and slot 0's tau: (Q online, Q target, a*, T, row loss, dtheta)."""
    theta = np.asarray(theta, F32)
    B = len(actions)
    R = B * per
    q0, q1 = q_values(theta[0, :R], per), q_values(theta[1, :R], per)
    astar = np.zeros(B, np.int64)
    T = np.zeros((B, per), F32)
    loss = np.zeros(B, F32)
    g = np.zeros((B, per), F32)
    for b in range(B):
        astar[b] = first_argmax(q1[b])
        rr, gam = returns[b]
        T[b] = QR.targets(rr, gam, theta[1, b * per:(b + 1) * per, astar[b]])
        loss[b], g[b] = loss_and_grad(T[b], theta[0, b * per:(b + 1) * per, int(actions[b])],
                                      tau0[b * per:(b + 1) * per], kappa, None if w is None else w[b])
    return q0, q1, astar, T, loss, g


def dz4(h4, w5_internal, actions, g, per):
    """Rule 10: (rows * per, 512) dZ4 from the online H4 rows, internal W5 (512, A) and dtheta (rows, per)."""
    h4 = np.asarray(h4, F32)
    col = np.asarray(w5_internal, F32)[:, np.repeat(np.asarray(actions), per)].T       # (R, 512)
    return np.where(h4 > 0, col * np.asarray(g, F32).reshape(-1, 1), F32(0)).astype(F32)


def fc2_grad(h4, actions, g, per, A):
    """Rule 10: fc2's gradient in Neon layout (A, 512), each column summed over its rows in row order."""
    h4 = np.asarray(h4, F32)
    gr = np.asarray(g, F32).reshape(-1)
    acts = np.repeat(np.asarray(actions), per)
    out = np.zeros((A, h4.shape[1]), F32)
    for r in range(h4.shape[0]):
        out[acts[r]] = out[acts[r]] + h4[r] * gr[r]
    return out


def mod_bwd(dx, ph, psi, per):
    """Rule 12: (dpsi (rows, cols), dphi (rows * per, cols))."""
    dx, ph, psi = np.asarray(dx, F32), np.asarray(ph, F32), np.asarray(psi, F32)
    rows = psi.shape[0]
    acc = np.zeros_like(psi)
    for j in range(per):
        acc = acc + dx[j::per][:rows] * ph[j::per][:rows]
    dpsi = np.where(psi > 0, acc, F32(0)).astype(F32)
    dphi = np.where(ph > 0, dx * np.repeat(psi, per, axis=0), F32(0)).astype(F32)
    return dpsi, dphi


def we_grad(c, dphi):
    """Rule 13: (64, cols) dWe, rows summed in order."""
    c, dphi = np.asarray(c, F32), np.asarray(dphi, F32)
    out = np.zeros((c.shape[1], dphi.shape[1]), F32)
    for r in range(c.shape[0]):
        out = out + c[r][:, None] * dphi[r][None, :]
    return out


def _conv_backward(weights, acts, d, n):
    """oracle.dqn_oracle.backward from the gradient at H3's flat (C, H, W) output down: grads of the three convs."""
    from oracle import dqn_oracle as O
    grads = [None] * 3
    for li in (2, 1, 0):
        r, s, k, st = O.CONV_GEOM[li]
        h_out = acts["h%d" % (li + 1)]
        _, _, p, q = h_out.shape
        d = d.reshape(n, k, p, q) * (h_out > 0)
        dz = np.ascontiguousarray(d.transpose(0, 2, 3, 1)).reshape(n * p * q, k)
        grads[li] = acts["cols%d" % li].T @ dz
        if li == 0:
            break
        x_in = acts["h%d" % li]
        c = x_in.shape[1]
        dcols = (dz @ weights[li].T).reshape(n, p, q, c, r, s)
        dx = np.zeros_like(x_in)
        for rr in range(r):
            for ss in range(s):
                dx[:, :, rr:rr + st * p:st, ss:ss + st * q:st] += dcols[:, :, :, :, rr, ss].transpose(0, 3, 1, 2)
        d = dx
    return grads


def forward(weights, states, tau):
    """The IQN network in Neon layout (weights[5] = We (3136, 64), rows in (c, p, q) order) on (B, ...) states at
    (B * per,) tau: (theta (B * per, A), activations for backward)."""
    from oracle import dqn_oracle as O
    _, acts = O.forward(weights[:5], states, keep=True)
    per = len(tau) // states.shape[0]
    c = cos_features(tau)
    ph = np.maximum(c @ weights[5].T, F32(0)).astype(F32)
    x = modulate(acts["flat"], ph, per)
    h4 = np.maximum(x @ weights[3].T, F32(0))
    acts.update(c=c, phi=ph, x=x, h4=h4, per=per)
    return (h4 @ weights[4].T).astype(F32), acts


def backward(weights, acts, deltas):
    """Gradients of all six layers (Neon layout) for (B * per, A) deltas on theta."""
    per, n = acts["per"], acts["flat"].shape[0]
    g4 = deltas.T @ acts["h4"]
    d = (deltas @ weights[4]) * (acts["h4"] > 0)
    g3 = d.T @ acts["x"]
    dx = d @ weights[3]
    ph, psi = acts["phi"], acts["flat"]
    dpsi = (dx * ph).reshape(n, per, -1).sum(axis=1) * (psi > 0)
    dphi = dx * np.repeat(psi, per, axis=0) * (ph > 0)
    g5 = dphi.T @ acts["c"]
    return [g.astype(F32) for g in _conv_backward(weights, acts, dpsi, n) + [g3, g4, g5]]


def numpy_step(weights, states, target_weights, minibatch, taus, kappa=1.0, discount=0.99, min_reward=-1,
               max_reward=1, lr=0.00025, decay=0.95):
    """One whole-network IQN step at the given (2, B * N) taus with RMSProp: the trajectory yardstick.  Updates weights /
    states in place; returns (cost, grads, T, dtheta)."""
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    B = len(actions)
    per = taus.shape[1] // B
    th_pre, acts = forward(weights, pre, taus[0])
    th_post, _ = forward(target_weights, post, taus[1])
    deltas = np.zeros_like(th_pre)
    T = np.zeros((B, per), F32)
    g = np.zeros((B, per), F32)
    cost = 0.0
    for b in range(B):
        a = int(actions[b])
        astar = first_argmax(q_values(th_post[b * per:(b + 1) * per], per)[0])
        rr, gam = one_step_return(rewards[b], terminals[b], discount, min_reward, max_reward)
        T[b] = QR.targets(rr, gam, th_post[b * per:(b + 1) * per, astar])
        l, g[b] = loss_and_grad(T[b], th_pre[b * per:(b + 1) * per, a], taus[0, b * per:(b + 1) * per], kappa)
        deltas[b * per:(b + 1) * per, a] = g[b]
        cost += float(l)
    grads = backward(weights, acts, deltas)
    O.rmsprop_update(weights, states, grads, B, lr=lr, decay=decay)
    return cost / B, grads, T, g
