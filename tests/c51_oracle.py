"""The distributional value head (C51, Bellemare, Dabney and Munos, 2017) on the CPU: a plain-Python and numpy
restatement of the device's k_fc2_dist, k_head_dist and k_opt_fc2_dist (csrc/net.cu), so that every output that does
not pass through expf / logf compares bit for bit when it is fed the device's own inputs.  A = actions, K = atoms.

Rules:
  1. Support (fp64): dz = (v_max - v_min) / (K - 1), z_i = v_min + i * dz; zf_i = float32(z_i).
  2. Logits: l[b][a * K + i] = sum_k H4[b][k] * W5[k][a * K + i], fp32, k = 0..511 in order, one rounding per product
     and per sum (no fused multiply-add).  W5 here is internal [512][A * K], i.e. the Neon weight transposed.
  3. Softmax per (slot, b, a) row, fp32: m = max_i l_i; e_i = exp(l_i - m); s = sum_i e_i in i order; p_i = e_i / s.
  4. Q[a] = sum_i zf_i * p_i, fp32, i order from 0.
  5. a* = first index of the maximum of slot 1's Q (slot 2's with Double DQN); q = p_slot1[a*].
  6. Return (fp64): R = clip(r) and g = gamma, or the n-step R and g = gamma^N (tests/nstep_oracle.py rule 3); g = 0
     when the window holds a terminal.
  7. Projection (fp64, j in order): T_j = min(max(R + g * z_j, v_min), v_max); b_j = (T_j - v_min) / dz;
     m_i = float32(sum_j q_j * max(0, 1 - |b_j - i|)).
  8. Loss: -(sum_i m_i * (l_i - m - log s)) at the taken action, fp32, i order; times the importance weight on a
     prioritized ring (td_err keeps the unweighted loss).
  9. gl_i = (p[a][i] - m_i), times the importance weight when there is one; 0 for the other actions.
 10. dZ4[k] = sum_i W5[k][a * K + i] * gl_i (fp32, i order) if H4[k] > 0 else 0; fp16 planes as the scalar head.
 11. dW5[k][a * K + i] = sum over the rows b whose action is a, in row order from 0, of H4_b[k] * gl_b,i.
 12. fc2's update: the configured optimizer of oracle/dqn_oracle.py on that gradient.
"""
import numpy as np

import nstep_oracle as NS

F32 = np.float32


def support(atoms, v_min, v_max):
    """Rule 1: (z fp64, zf float32, dz)."""
    dz = (float(v_max) - float(v_min)) / (atoms - 1)
    z = np.array([float(v_min) + i * dz for i in range(atoms)], np.float64)
    return z, z.astype(F32), dz


def logits(h4, w5_internal):
    """Rule 2 for a (rows, 512) H4 and an internal (512, A*K) W5."""
    h4 = np.asarray(h4, F32)
    w5 = np.asarray(w5_internal, F32)
    acc = np.zeros((h4.shape[0], w5.shape[1]), F32)
    for k in range(h4.shape[1]):
        acc = acc + h4[:, k:k + 1] * w5[k:k + 1, :]
    return acc


def softmax(l):
    """Rule 3 on the last axis (numpy's float32 exp: within CUDA's expf bound of the device, not bit for bit)."""
    l = np.asarray(l, F32)
    m = l.max(axis=-1, keepdims=True)
    e = np.exp(l - m).astype(F32)
    s = np.zeros(l.shape[:-1] + (1,), F32)
    for i in range(l.shape[-1]):
        s = s + e[..., i:i + 1]
    return e / s


def q_values(p, zf):
    """Rule 4 on the last axis."""
    p = np.asarray(p, F32)
    q = np.zeros(p.shape[:-1], F32)
    for i in range(p.shape[-1]):
        q = q + zf[i] * p[..., i]
    return q


def first_argmax(q):
    best = 0
    for j in range(1, len(q)):
        if q[j] > q[best]:
            best = j
    return best


def one_step_return(r, terminal, discount, min_reward=-1, max_reward=1):
    """Rule 6 at N = 1: (R, g)."""
    return NS.clip_reward(r, min_reward, max_reward), 0.0 if terminal else float(discount)


def n_step_return(rewards, terminals, discount, min_reward=-1, max_reward=1):
    """Rule 6: (R, g)."""
    R, g, term = NS.n_step_return(rewards, terminals, discount, min_reward, max_reward)
    return R, 0.0 if term else g


def project(R, g, q, z, v_min, v_max, dz):
    """Rule 7: the target distribution m (float32) of one sample."""
    atoms = len(z)
    b = []
    for j in range(atoms):
        T = min(max(R + g * float(z[j]), float(v_min)), float(v_max))
        b.append((T - float(v_min)) / dz)
    m = np.zeros(atoms, F32)
    for i in range(atoms):
        acc = 0.0
        for j in range(atoms):
            acc = acc + float(q[j]) * max(0.0, 1.0 - abs(b[j] - i))
        m[i] = F32(acc)
    return m


def loss(m, l_row):
    """Rule 8 for one sample (float32 log: within CUDA's logf bound of the device)."""
    l_row = np.asarray(l_row, F32)
    mx = l_row.max()
    s = F32(0)
    for v in np.exp(l_row - mx).astype(F32):
        s = F32(s + v)
    ls = F32(np.log(s))
    acc = F32(0)
    for i in range(len(m)):
        acc = F32(acc + F32(m[i]) * F32(F32(l_row[i] - mx) - ls))
    return F32(-acc)


def logit_grad(p_row, m, w=None):
    """Rule 9 at the taken action."""
    g = (np.asarray(p_row, F32) - np.asarray(m, F32)).astype(F32)
    return g if w is None else (g * F32(w)).astype(F32)


def dz4(h4_row, w5_internal, a, gl):
    """Rule 10 for one sample."""
    K = len(gl)
    blk = np.asarray(w5_internal, F32)[:, a * K:(a + 1) * K]
    acc = np.zeros(blk.shape[0], F32)
    for i in range(K):
        acc = acc + blk[:, i] * F32(gl[i])
    return np.where(np.asarray(h4_row) > 0, acc, F32(0)).astype(F32)


def fp16_planes(d):
    """The hi / scaled-lo fp16 planes of a dZ4 row, as every head writes them."""
    hi = np.asarray(d, F32).astype(np.float16)
    lo = ((np.asarray(d, F32) - hi.astype(F32)) * F32(2048)).astype(np.float16)
    return hi, lo


def fc2_grad(h4, gl, actions, num_actions):
    """Rule 11: dW5 in Neon layout (A*K, 512)."""
    h4, gl = np.asarray(h4, F32), np.asarray(gl, F32)
    K = gl.shape[1]
    g = np.zeros((num_actions * K, h4.shape[1]), F32)
    for a in range(num_actions):
        acc = np.zeros((K, h4.shape[1]), F32)
        for b in range(h4.shape[0]):
            if actions[b] == a:
                acc = acc + gl[b][:, None] * h4[b][None, :]
        g[a * K:(a + 1) * K] = acc
    return g


def head(probs, actions, returns, z, v_min, v_max, dz, double=False, w=None):
    """Rules 5, 7 and 9 on the device's (3, batch, A, K) probabilities and per-sample (R, g): (a*, m, gl)."""
    probs = np.asarray(probs, F32)
    zf = z.astype(F32)
    n = len(actions)
    astar = np.zeros(n, np.int64)
    m = np.zeros((n, len(z)), F32)
    gl = np.zeros((n, len(z)), F32)
    for b in range(n):
        q_sel = q_values(probs[2 if double else 1, b], zf)
        astar[b] = first_argmax(q_sel)
        R, g = returns[b]
        m[b] = project(R, g, probs[1, b, astar[b]], z, v_min, v_max, dz)
        gl[b] = logit_grad(probs[0, b, actions[b]], m[b], None if w is None else w[b])
    return astar, m, gl


def numpy_step(weights, states, target_weights, minibatch, atoms, v_min, v_max, discount=0.99, min_reward=-1,
               max_reward=1, lr=0.00025, decay=0.95):
    """One whole-network C51 step in numpy (oracle.dqn_oracle's forward, backward and RMSProp with this head): the
    trajectory yardstick.  Updates weights / states (RMSProp planes) in place; returns (cost, grads, m, gl)."""
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    z, zf, dz = support(atoms, v_min, v_max)
    l_pre, acts = O.forward(weights, pre, keep=True)             # (B, A*K): H4 @ W5^T
    l_post = O.forward(target_weights, post)
    B = len(actions)
    A = l_pre.shape[1] // atoms
    p_pre = softmax(l_pre.reshape(B, A, atoms))
    p_post = softmax(l_post.reshape(B, A, atoms))
    deltas = np.zeros((B, A * atoms), F32)
    m = np.zeros((B, atoms), F32)
    gl = np.zeros((B, atoms), F32)
    cost = 0.0
    for b in range(B):
        a = int(actions[b])
        astar = first_argmax(q_values(p_post[b], zf))
        R, g = one_step_return(rewards[b], terminals[b], discount, min_reward, max_reward)
        m[b] = project(R, g, p_post[b, astar], z, v_min, v_max, dz)
        gl[b] = logit_grad(p_pre[b, a], m[b])
        deltas[b, a * atoms:(a + 1) * atoms] = gl[b]
        cost += float(loss(m[b], l_pre[b, a * atoms:(a + 1) * atoms]))
    grads = O.backward(weights, acts, deltas)
    O.rmsprop_update(weights, states, grads, B, lr=lr, decay=decay)
    return cost / B, grads, m, gl
