"""The Munchausen DQN target (M-DQN, Vieillard, Pietquin and Geist, 2020) on the CPU: a numpy restatement of the target
k_head_mdqn forms (csrc/net.cu), and a whole-network numpy Munchausen step.  The rest of the head (delta, clip, cost,
dZ4, fc2's gradient) is the scalar head's (tests/head_oracle.py).  Every fp64 operation is rounded on its own (Python
floats), except exp and log: the device's fp64 functions are not bit-identical to the C library's, so a device target
is held within one fp32 ulp of this one, not bit for bit.

Rules (include/b200dqn.h states them too), for a sample with taken action a:
  1. Per fp32 row x (the target network's Q on the poststates, and on the prestates): m = max_j x_j;
     e_j = exp((double(x_j) - m) / tau); s = sum_j e_j in j order; lse = m + tau * log(s); lp_j = double(x_j) - lse
     (tau ln pi_j); pi_j = e_j / s.
  2. bonus = alpha * min(max(lp_pre[a], l0), 0).
  3. next = sum_j pi_post,j * (x_post,j - lp_post,j) in j order.
  4. y = (R + bonus) + g * next, R the clipped (or n-step) return, g = gamma (gamma^N), 0 when the window holds a
     terminal (then y = R + bonus).  The last operation is the scalar head's: one fused multiply-add on the one-step
     step (the SASS of k_head<2, false> and k_head_mdqn<., false> contracts it into a DFMA), a separately rounded
     product and sum on the n-step step.
  5. target = float32(y).
"""
import math
from fractions import Fraction

import numpy as np

import c51_oracle as C51

F32 = np.float32
one_step_return = C51.one_step_return
n_step_return = C51.n_step_return


def fma(a, b, c):
    """a * b + c rounded once (math.fma is Python 3.13+)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def row_stats(x, tau):
    """Rule 1 on one fp32 row: (lp, pi) as lists of Python floats."""
    x = [float(v) for v in np.asarray(x, F32)]
    m = max(x)
    e = [math.exp((v - m) / tau) for v in x]
    s = 0.0
    for v in e:
        s += v
    lse = m + tau * math.log(s)
    return [v - lse for v in x], [v / s for v in e]


def bonus(x_pre, a, alpha, tau, l0):
    """Rule 2."""
    lp, _ = row_stats(x_pre, tau)
    return alpha * min(max(lp[a], l0), 0.0)


def soft_value(x_post, tau):
    """Rule 3."""
    lp, pi = row_stats(x_post, tau)
    nxt = 0.0
    for xj, lj, pj in zip(np.asarray(x_post, F32), lp, pi):
        nxt += pj * (float(xj) - lj)
    return nxt


def target64(x_post, x_pre, a, R, g, alpha, tau, l0, nstep=False):
    """Rules 1-4: y as a Python float.  g = 0 marks a terminal."""
    rb = R + bonus(x_pre, a, alpha, tau, l0)
    if g == 0:
        return rb
    nxt = soft_value(x_post, tau)
    return rb + g * nxt if nstep else fma(g, nxt, rb)


def scalar_y(maxq, R, g, nstep=False):
    """The scalar head's y on the same operands (k_head): the yardstick of the one-action identity."""
    if g == 0:
        return R
    return R + g * float(F32(maxq)) if nstep else fma(g, float(F32(maxq)), R)


def targets(q_post, q_pre, actions, returns, alpha, tau, l0, nstep=False):
    """Rule 5 over a batch: float32 targets from the device's (batch, A) rows and per-sample (R, g)."""
    return np.array([F32(target64(q_post[b], q_pre[b], int(actions[b]), returns[b][0], returns[b][1], alpha, tau, l0,
                                  nstep)) for b in range(len(actions))], F32)


def numpy_step(weights, states, target_weights, minibatch, alpha=0.9, tau=0.03, l0=-1.0, discount=0.99, min_reward=-1,
               max_reward=1, clip=1.0, lr=0.00025, decay=0.95):
    """One whole-network Munchausen step in numpy (oracle.dqn_oracle's forward, backward and RMSProp with this target):
    the trajectory yardstick.  Updates weights / states (RMSProp planes) in place; returns (cost, grads, y)."""
    from oracle import dqn_oracle as O
    pre, actions, rewards, post, terminals = minibatch
    preq, acts = O.forward(weights, pre, keep=True)
    q_post = O.forward(target_weights, post)
    q_pre = O.forward(target_weights, pre)
    B = len(actions)
    returns = [one_step_return(rewards[b], terminals[b], discount, min_reward, max_reward) for b in range(B)]
    y = targets(q_post, q_pre, actions, returns, alpha, tau, l0)
    deltas = np.zeros_like(preq)
    cost = 0.0
    for b in range(B):
        a = int(actions[b])
        d = F32(preq[b, a] - y[b])
        cost += float(F32(0.5) * d * d)
        deltas[b, a] = np.clip(d, -clip, clip) if clip else d
    grads = O.backward(weights, acts, deltas.astype(F32))
    O.rmsprop_update(weights, states, grads, B, lr=lr, decay=decay)
    return cost / B, grads, y
