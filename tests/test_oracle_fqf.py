"""CPU checks of tests/fqf_oracle.py, the restatement the GPU tests hold the FQF head to: the fraction gradient against
finite differences of the Wasserstein-1 error of an analytic quantile function, the chain g -> dl -> dW_f against torch
autograd in float64, the uniform proposal of zero logits, and the creation refusals, which fire ahead of any device
work."""
import ctypes as C

import numpy as np
import pytest
from scipy import integrate

import fqf_oracle as FQ

F32 = np.float32


def _finv(w):
    """An analytic, strictly increasing quantile function on (0, 1)."""
    return np.log(w / (1.0 - w)) + 2.0 * w ** 3


def _w1(tau):
    """sum_i int_{tau_i}^{tau_{i+1}} |F^-1(w) - F^-1(tauhat_i)| dw, tauhat_i the midpoint, in float64."""
    total = 0.0
    for i in range(len(tau) - 1):
        lo, hi = tau[i], tau[i + 1]
        c = _finv(0.5 * (lo + hi))
        total += integrate.quad(lambda w: abs(_finv(w) - c), lo, hi, points=[0.5 * (lo + hi)], epsabs=1e-13,
                                epsrel=1e-12, limit=200)[0]
    return total


@pytest.mark.parametrize("N", [2, 3, 8])
def test_fraction_gradient_is_the_w1_derivative(N):
    """Rule 7's g_i (theta = F^-1 at tauhat, beta = F^-1 at tau_i) against central differences of W1 in each interior
    tau_i (tau_0 = 0 and tau_N = 1 fixed; the ends stay away from F^-1's poles)."""
    rs = np.random.RandomState(N)
    inner = np.sort(rs.uniform(0.05, 0.95, N - 1))
    tau = np.concatenate([[1e-3], inner, [1 - 1e-3]])
    tauhat = 0.5 * (tau[:-1] + tau[1:])
    theta_a = _finv(tauhat)[None]
    beta = _finv(tau[1:-1])[None]
    g, _ = FQ.fraction_grads(theta_a, beta, np.full((1, N), 1.0 / N), dtype=np.float64)
    h = 1e-5
    for i in range(1, N):
        tp, tm = tau.copy(), tau.copy()
        tp[i] += h
        tm[i] -= h
        fd = (_w1(tp) - _w1(tm)) / (2 * h)
        assert abs(g[0, i - 1] - fd) <= 1e-5 * max(1.0, abs(fd)), (i, g[0, i - 1], fd)


@pytest.mark.parametrize("weighted", [False, True])
def test_logit_and_layer_gradients_match_autograd(weighted):
    """g -> dl -> dW_f (rules 2, 7, 8 in fp32) against float64 torch autograd of sum_b sum_i g_bi tau_bi(l_b), g
    detached, l_b = W_f psi_b: dl within a relative L2 error of 1e-5, dW_f within 1e-4."""
    import torch
    rs = np.random.RandomState(3)
    B, N, cols = 6, 8, 3136
    psi = np.maximum(rs.randn(B, cols), 0).astype(F32)
    wf = (rs.randn(N, cols) * 0.01).astype(F32)
    l = FQ.logits(psi, wf)
    q, tau, tauhat = FQ.proposal(l)
    theta_a = np.sort(rs.randn(B, N), axis=1).astype(F32)
    beta = (0.5 * (theta_a[:, 1:] + theta_a[:, :-1]) + 0.1 * rs.randn(B, N - 1)).astype(F32)
    w = rs.uniform(0.2, 1.0, B).astype(F32) if weighted else None
    g, dl = FQ.fraction_grads(theta_a, beta, q, w)
    dwf = FQ.wf_grad(dl, psi)
    W = torch.tensor(wf.astype(np.float64), requires_grad=True)
    lt = torch.tensor(psi.astype(np.float64)) @ W.T
    lt.retain_grad()
    taus = torch.cumsum(torch.softmax(lt, dim=1), dim=1)[:, :N - 1]      # tau_1 .. tau_{N-1}
    (torch.tensor(g.astype(np.float64)) * taus).sum().backward()
    rel = lambda a, b: float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))
    assert rel(dl.astype(np.float64), lt.grad.numpy()) <= 1e-5
    assert rel(dwf.astype(np.float64), W.grad.numpy()) <= 1e-4
    # the restated fp64 proposal agrees with torch's softmax
    assert np.allclose(q, torch.softmax(torch.tensor(l.astype(np.float64)), 1).numpy(), rtol=1e-6, atol=1e-9)
    assert (tau[:, 0] == 0).all() and (tau[:, -1] == 1).all() and (np.diff(tau, axis=1) >= 0).all()
    assert ((tauhat > tau[:, :-1]) & (tauhat < tau[:, 1:])).all()


@pytest.mark.parametrize("N", [2, 3, 8, 32, 64])
def test_zero_logits_give_the_qr_midpoints(N):
    q, tau, tauhat = FQ.proposal(np.zeros((3, N), F32))
    assert (tauhat == FQ.midpoints(N)[None]).all()
    assert (tau[:, 0] == 0).all() and (tau[:, -1] == 1).all()
    assert (q == F32(1.0 / N)).all()


def test_logit_order_and_q_rule():
    """Rule 1's lane order is a fixed fp32 order close to the float64 dot product; rule 4 with equal fractions is the
    mean up to rounding, and with one action picks action 0."""
    rs = np.random.RandomState(5)
    psi = np.maximum(rs.randn(4, 3136), 0).astype(F32)
    wf = rs.randn(5, 3136).astype(F32) * F32(0.02)
    l = FQ.logits(psi, wf)
    assert np.allclose(l, psi.astype(np.float64) @ wf.T.astype(np.float64), rtol=1e-5, atol=1e-5)
    _, tau, tauhat = FQ.proposal(np.zeros((4, 8), F32))
    theta = rs.randn(2, 32, 3).astype(F32)
    q = FQ.q_values(theta[0], tau)
    assert np.allclose(q, theta[0].reshape(4, 8, 3).mean(axis=1), rtol=1e-6, atol=1e-6)
    th1 = rs.randn(2, 8, 1).astype(F32)
    _, tau1, tauhat1 = FQ.proposal(np.zeros((1, 8), F32))
    _, _, astar, _, _, _ = FQ.head(th1, tauhat1[0], tau1, [0], [(0.0, 0.99)], 1.0)
    assert astar[0] == 0


def test_net_create_refuses_before_device_work():
    """num_fractions outside {0} and 2..64, more than 4096 rows, a bad fraction_lr, a second head or a non-finite
    clip_error are EINVAL; dueling and Munchausen are ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.num_fractions == 0 and cfg.fraction_lr == 2.5e-9
    for fields, exc, match in (({"num_fractions": -1}, AssertionError, "num_fractions"),
                               ({"num_fractions": 1}, AssertionError, "num_fractions"),
                               ({"num_fractions": 65}, AssertionError, "num_fractions"),
                               ({"batch_size": 65, "num_fractions": 64}, AssertionError, "4096"),
                               ({"batch_size": 2049, "num_fractions": 2}, AssertionError, "4096"),
                               ({"fraction_lr": -1e-9}, AssertionError, "fraction_lr"),
                               ({"fraction_lr": float("nan")}, AssertionError, "fraction_lr"),
                               ({"fraction_lr": float("inf")}, AssertionError, "fraction_lr"),
                               ({"num_atoms": 51}, AssertionError, "one"),
                               ({"num_quantiles": 8}, AssertionError, "one"),
                               ({"num_tau_samples": 8}, AssertionError, "one"),
                               ({"num_heads": 4}, AssertionError, "one"),
                               ({"clip_error": float("inf")}, AssertionError, "clip_error"),
                               ({"dueling": 1}, NotImplementedError, "FQF"),
                               ({"munchausen": 1}, NotImplementedError, "FQF")):
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.num_fractions = 8
        for k, v in fields.items():
            setattr(cfg, k, v)
        with pytest.raises(exc, match=match):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
