"""CPU checks of tests/munchausen_oracle.py, the restatement the GPU tests hold the Munchausen target to: its rules
against an independent float64 statement of the paper's formula (scipy's logsumexp and softmax), its limits (one
action, l0 = 0, alpha = 0 with tau -> 0), a whole-network numpy step against torch autograd, and the creation
refusals, which fire ahead of any device work."""
import ctypes as C

import numpy as np
import pytest

import munchausen_oracle as M

F32 = np.float32


def _paper(q_post, q_pre, a, R, g, alpha, tau, l0):
    """y = R + alpha clip(tau log pi(a|s), l0, 0) + g sum_a' pi(a'|s') (q(s', a') - tau log pi(a'|s')), float64."""
    from scipy.special import log_softmax, softmax
    qo, qp = np.asarray(q_post, np.float64), np.asarray(q_pre, np.float64)
    lp_pre = tau * log_softmax(qp / tau)
    lp_post = tau * log_softmax(qo / tau)
    nxt = float((softmax(qo / tau) * (qo - lp_post)).sum())
    return R + alpha * min(max(float(lp_pre[a]), l0), 0.0) + g * nxt, nxt


def _rows(A, spread, seed):
    rs = np.random.RandomState(seed)
    return (rs.randn(A) * spread).astype(F32), (rs.randn(A) * spread + 0.1).astype(F32)


@pytest.mark.parametrize("A", [1, 2, 18, 32])
@pytest.mark.parametrize("tau", [1e-3, 0.03, 1.0])
def test_rules_match_the_paper(A, tau):
    """Every alpha, l0, terminal and n-step case within 1e-12 of the paper's formula in float64, relative to the size
    of the terms (the rules and scipy take different but each accurate paths to the log-policy)."""
    for seed in range(4):
        for spread in (0.5, 5.0):
            q_post, q_pre = _rows(A, spread, seed)
            a = seed % A
            for alpha in (0.0, 0.9, 1.0):
                for l0 in (-1.0, 0.0):
                    for R, g, nstep in ((0.5, 0.99, False), (-1.0, 0.0, False), (1.75, 0.99 ** 3, True),
                                        (-0.5, 0.0, True)):
                        y = M.target64(q_post, q_pre, a, R, g, alpha, tau, l0, nstep)
                        ref, nxt = _paper(q_post, q_pre, a, R, g, alpha, tau, l0)
                        scale = abs(R) + alpha + abs(g) * (abs(nxt) + np.abs(q_post).max() + tau * np.log(A) + 1)
                        assert abs(y - ref) <= 1e-12 * scale, (seed, alpha, l0, R, g, y, ref)


def test_wide_spreads_stay_finite():
    """Q spreads of 100 at tau = 0.03 (exponents down to -3333): no overflow, NaN or -inf, and still the paper's
    value; the bonus saturates at l0."""
    for A in (2, 18, 32):
        for seed in range(3):
            q_post, q_pre = _rows(A, 1.0, seed)
            q_post[0], q_pre[1] = F32(100), F32(-100)
            for a in range(A):
                y = M.target64(q_post, q_pre, a, 1.0, 0.99, 0.9, 0.03, -1.0)
                ref, nxt = _paper(q_post, q_pre, a, 1.0, 0.99, 0.9, 0.03, -1.0)
                assert np.isfinite(y) and abs(y - ref) <= 1e-12 * (2 + 100 + abs(nxt)), (A, seed, a, y, ref)
            assert M.bonus(q_pre, 1, 0.9, 0.03, -1.0) == -0.9


@pytest.mark.parametrize("nstep", [False, True])
def test_one_action_is_the_scalar_head(nstep):
    """A = 1: pi = 1, tau ln pi = 0 exactly, so the bonus is 0 and next is the lone Q value: y is k_head's y bit for
    bit, for any alpha, tau and l0."""
    rs = np.random.RandomState(1)
    for _ in range(200):
        q_post, q_pre = (rs.randn(1) * 10).astype(F32), (rs.randn(1) * 10).astype(F32)
        R, g = float(rs.randint(-1, 2)), [0.0, 0.99, 0.97 ** 3][rs.randint(3)]
        for alpha, tau, l0 in ((0.9, 0.03, -1.0), (1.0, 1e-3, 0.0), (0.0, 1.0, -5.0)):
            assert M.target64(q_post, q_pre, 0, R, g, alpha, tau, l0, nstep) == M.scalar_y(q_post[0], R, g, nstep)


def test_l0_zero_removes_the_bonus():
    """tau ln pi <= 0, so clamp(., 0, 0) = 0: the target is the soft (entropy-regularised) one with no bonus."""
    for seed in range(5):
        q_post, q_pre = _rows(18, 2.0, seed)
        for a in range(18):
            assert M.bonus(q_pre, a, 0.9, 0.03, 0.0) == 0
            y = M.target64(q_post, q_pre, a, 0.5, 0.99, 0.9, 0.03, 0.0)
            assert y == M.target64(q_post, q_pre, a, 0.5, 0.99, 0.0, 0.03, -1.0)


def test_hard_limit_is_the_dqn_target():
    """alpha = 0 and every Q gap above 746 tau (exp underflows to exactly 0): pi is one-hot at the maximum, next is
    max_a Q, and y is the DQN y bit for bit."""
    rs = np.random.RandomState(3)
    for A in (2, 18, 32):
        for tau in (1e-3, 0.03):
            q_post = (np.arange(A) * 800 * tau + rs.rand() * 0.1).astype(F32)
            rs.shuffle(q_post)
            q_pre = rs.randn(A).astype(F32)
            for nstep in (False, True):
                y = M.target64(q_post, q_pre, 0, 0.5, 0.99, 0.0, tau, -1.0, nstep)
                assert y == M.scalar_y(q_post.max(), 0.5, 0.99, nstep), (A, tau, nstep)


def test_rules_are_sensitive_to_their_mutations():
    """The mutations the device tests must catch each move y by far more than one fp32 ulp: the log-policy's sign, the
    clamp dropped, the bonus cut at terminals, tau left out of the lse."""
    q_post, q_pre = _rows(4, 3.0, 7)
    a, R, g, alpha, tau, l0 = int(np.argmin(q_pre)), 0.5, 0.99, 0.9, 0.03, -1.0
    y = M.target64(q_post, q_pre, a, R, g, alpha, tau, l0)
    lp, _ = M.row_stats(q_pre, tau)
    ulp = float(np.spacing(F32(y)))
    assert lp[a] < l0                                                  # the clamp is live in this case
    assert abs(alpha * min(max(-lp[a], l0), 0.0) - alpha * min(max(lp[a], l0), 0.0)) > 100 * ulp
    assert abs(alpha * lp[a] - alpha * l0) > 100 * ulp
    assert abs(M.target64(q_post, q_pre, a, R, 0.0, alpha, tau, l0) - R) > 100 * ulp
    close = (q_post * F32(0.01)).astype(F32)                            # a row whose soft-max is not one-hot
    m = float(close.max())
    s = sum(np.exp((float(v) - m) / tau) for v in close)
    assert abs((m + np.log(s)) - (m + tau * np.log(s))) > 100 * ulp


def test_numpy_step_matches_torch_autograd_of_the_whole_network():
    """The numpy Munchausen step's gradients of all five layers equal torch autograd of sum_b huber(q(s_b, a_b) -
    stop_grad(y_b)) (Huber threshold clip_error, whose gradient is the clipped delta) through the whole network in
    float64, with y from the target network held fixed."""
    torch = pytest.importorskip("torch")
    from oracle import dqn_oracle as O
    A, B = 4, 4
    rs = np.random.RandomState(2)
    ws = [np.asarray(w, F32) for w in O.xavier_init(A, 5)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.1) * np.abs(w).max()).astype(F32) for w in ws]
    pre = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    act = rs.randint(0, A, B)
    rew = np.array([1, -1, 0, 2])
    term = np.array([False, True, False, False])
    for clip in (1.0, 0.0):
        wk = [w.copy() for w in ws]
        _, grads, y = M.numpy_step(wk, [np.zeros_like(w) for w in wk], tws, (pre, act, rew, post, term), clip=clip)
        tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in ws]
        h = torch.from_numpy(pre).double() / 255.0
        for li, (r, s_, k, st) in enumerate(O.CONV_GEOM):
            w = tw[li].reshape(h.shape[1], r, s_, k).permute(3, 0, 1, 2)
            h = torch.relu(torch.nn.functional.conv2d(h, w, stride=st))
        q = torch.relu(h.flatten(1) @ tw[3].T) @ tw[4].T
        d = q[torch.arange(B), torch.tensor(act)] - torch.tensor(y, dtype=torch.float64)
        loss = torch.where(d.abs() <= clip, 0.5 * d * d, clip * (d.abs() - 0.5 * clip)) if clip else 0.5 * d * d
        loss.sum().backward()
        assert np.abs(y).max() > 0
        for layer in range(5):
            ref = tw[layer].grad.numpy()
            err = np.linalg.norm(grads[layer] - ref) / max(np.linalg.norm(ref), 1e-30)
            assert err <= 1e-4, (clip, layer, err)


def test_net_create_refuses_before_device_work():
    """munchausen outside {0, 1}, a non-finite or negative alpha, a non-finite or non-positive tau and a non-finite or
    positive l0 are EINVAL; with the dueling network or a distributional or quantile head it is ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert (cfg.munchausen, cfg.munchausen_alpha, cfg.munchausen_tau, cfg.munchausen_clip) == (0, 0.9, 0.03, -1.0)
    inf, nan = float("inf"), float("nan")
    cases = [({"munchausen": 2}, AssertionError), ({"munchausen": -1}, AssertionError)]
    cases += [({"munchausen_alpha": v}, AssertionError) for v in (-0.1, inf, nan)]
    cases += [({"munchausen_tau": v}, AssertionError) for v in (0.0, -0.03, inf, nan)]
    cases += [({"munchausen_clip": v}, AssertionError) for v in (0.5, -inf, nan)]
    cases += [({"dueling": 1}, NotImplementedError), ({"num_atoms": 51}, NotImplementedError),
              ({"num_quantiles": 51}, NotImplementedError)]
    for fields, exc in cases:
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.munchausen = 1
        for k, v in fields.items():
            setattr(cfg, k, v)
        with pytest.raises(exc, match="Munchausen"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
