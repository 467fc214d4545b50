"""The fully parameterized quantile function head (FQF, Yang, Zhao, Lin, Qin, Bian and Liu, 2019) on the CPU: a numpy
restatement of the device's k_fqf_fraction, k_head_fqf and k_fqf_wf (csrc/net.cu), so that every output compares bit for
bit when it is fed the device's own inputs.  The rest of the network (c, phi, X, fc1, fc2, the quantile loss and its
backward) is the IQN head's, tests/iqn_oracle.py, at tau = tauhat.  N = num_fractions, b the sample, a the taken action,
psi the online network's H3 of the prestates.  Every operation is fp32 with its own rounding unless marked fp64.

Rules (include/b200dqn.h states them too):
  1. l[b][k] = sum_col psi[b][col] W_f[k][col] over fc1's internal columns: 32 lanes, lane j sums columns j, j + 32, ...
     in order, then the lanes are combined by halving (s_j += s_{j + h}, h = 16, 8, 4, 2, 1).
  2. fp64: e_k = exp(l_k - max l); C_{i+1} = C_i + e_i; S = C_N; q_k = float(e_k / S); tau_i = float(C_i / S);
     tauhat_i = float((C_i + C_{i+1}) / 2S) (numpy's exp: within one fp32 ulp of the device, not bit for bit).
  4. Q[a] = sum_i (tau_{i+1} - tau_i) theta[b N + i][a], i order.
  5. The quantile loss and dtheta are the IQN head's with weights tauhat.
  7. g_i = (2 beta_i - theta[b N + i][a]) - theta[b N + i - 1][a] (times w_b); dq_k = sum_{i > k} g_i from i = N - 1
     down; s = sum_k q_k dq_k; dl_k = q_k (dq_k - s).
  8. dW_f[k][col] = sum_b dl[b][k] psi[b][col], b order.
"""
import numpy as np

import iqn_oracle as IQ
import qr_oracle as QR

F32 = np.float32
FLAT = 3136

first_argmax = IQ.first_argmax
one_step_return = IQ.one_step_return
n_step_return = IQ.n_step_return


def logits(psi, wf):
    """Rule 1: (B, N) from psi (B, 3136) and W_f (N, 3136), both in fc1's internal column order."""
    psi, wf = np.asarray(psi, F32), np.asarray(wf, F32)
    prod = psi[:, None, :] * wf[None, :, :]                     # (B, N, 3136), each product rounded
    lanes = np.zeros(prod.shape[:2] + (32,), F32)
    for i in range(FLAT // 32):
        lanes = lanes + prod[:, :, 32 * i:32 * (i + 1)]
    h = 16
    while h:
        lanes = lanes[..., :h] + lanes[..., h:2 * h]
        h //= 2
    return lanes[..., 0].astype(F32)


def proposal(l):
    """Rule 2: (q (B, N), tau (B, N + 1), tauhat (B, N)) float32 from (B, N) logits."""
    l = np.asarray(l, F32).astype(np.float64)
    B, N = l.shape
    m = l.max(axis=1, keepdims=True)
    e = np.exp(l - m)
    C = np.zeros((B, N + 1))
    for k in range(N):
        C[:, k + 1] = C[:, k] + e[:, k]
    S = C[:, N:N + 1]
    q = (e / S).astype(F32)
    tau = (C / S).astype(F32)
    tauhat = ((C[:, :N] + C[:, 1:]) / (2.0 * S)).astype(F32)
    return q, tau, tauhat


def q_values(theta_rows, tau):
    """Rule 4: (B, A) Q from (B N, A) theta and (B, N + 1) fractions."""
    tau = np.asarray(tau, F32)
    B, N = tau.shape[0], tau.shape[1] - 1
    th = np.asarray(theta_rows, F32)[:B * N].reshape(B, N, -1)
    dt = (tau[:, 1:] - tau[:, :-1]).astype(F32)
    q = np.zeros((B, th.shape[2]), F32)
    for i in range(N):
        q = q + dt[:, i:i + 1] * th[:, i]
    return q


def head(theta, tauhat0, tau, actions, returns, kappa, w=None):
    """Rules 4 and 5 on the device's (2, >= B N, A) theta: (Q online, Q target, a*, T, row loss, dtheta)."""
    theta, tau = np.asarray(theta, F32), np.asarray(tau, F32)
    B, N = tau.shape[0], tau.shape[1] - 1
    q0, q1 = q_values(theta[0], tau), q_values(theta[1], tau)
    astar = np.zeros(B, np.int64)
    T = np.zeros((B, N), F32)
    loss = np.zeros(B, F32)
    g = np.zeros((B, N), F32)
    for b in range(B):
        astar[b] = first_argmax(q1[b])
        rr, gam = returns[b]
        T[b] = QR.targets(rr, gam, theta[1, b * N:(b + 1) * N, astar[b]])
        loss[b], g[b] = IQ.loss_and_grad(T[b], theta[0, b * N:(b + 1) * N, int(actions[b])],
                                         tauhat0[b * N:(b + 1) * N], kappa, None if w is None else w[b])
    return q0, q1, astar, T, loss, g


def fraction_grads(theta_a, beta, q, w=None, dtype=F32):
    """Rule 7: (g (B, N - 1), dl (B, N)) from theta at tauhat of the taken action (B, N), beta (B, N - 1) and q (B, N),
    in `dtype` (float64 for the finite-difference check)."""
    th, beta, q = (np.asarray(x, dtype) for x in (theta_a, beta, q))
    B, N = th.shape
    g = (dtype(2) * beta - th[:, 1:]) - th[:, :-1]
    if w is not None:
        g = g * np.asarray(w, dtype)[:, None]
    dq = np.zeros((B, N), dtype)
    acc = np.zeros(B, dtype)
    for k in range(N - 2, -1, -1):
        acc = acc + g[:, k]                          # g[:, k] is g_{k+1}
        dq[:, k] = acc
    s = np.zeros(B, dtype)
    for k in range(N):
        s = s + q[:, k] * dq[:, k]
    dl = q * (dq - s[:, None])
    return g.astype(dtype), dl.astype(dtype)


def wf_grad(dl, psi):
    """Rule 8: (N, cols) dW_f, samples summed in order."""
    dl, psi = np.asarray(dl, F32), np.asarray(psi, F32)
    out = np.zeros((dl.shape[1], psi.shape[1]), F32)
    for b in range(dl.shape[0]):
        out = out + dl[b][:, None] * psi[b][None, :]
    return out


def midpoints(N):
    """The quantile-regression head's fixed fractions float((2i + 1) / 2N)."""
    return np.array([(2 * i + 1) / (2 * N) for i in range(N)], dtype=np.float64).astype(F32)
