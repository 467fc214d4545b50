"""CPU checks of tests/iqn_oracle.py, the restatement the GPU tests hold the IQN head to: the tau generator (its hash,
the open interval, exact complements), the whole-network numpy step against torch autograd in float64 (embedding
included), the limits (a constant embedding, one action), and the creation refusals, which fire ahead of any device
work."""
import ctypes as C

import numpy as np
import pytest

import iqn_oracle as IQ

F32 = np.float32


def test_tau_generator_is_the_stated_hash():
    """splitmix64's finaliser at a known input (the reference value of its published test vector), then the draw."""
    assert IQ._mix(0x9E3779B97F4A7C15) == 0xE220A8397B1DCDAF
    t = IQ.tau_draw(12345, 7, 2, 64, 64)
    assert (t > 0).all() and (t < 1).all()
    m = t.astype(np.float64) * 2.0 ** 24
    assert (m == np.round(m)).all() and (np.round(m) % 2 == 1).all()      # (2m + 1) 2^-24, exact in fp32
    assert ((F32(1) - t).astype(np.float64) == 1.0 - t.astype(np.float64)).all()
    assert len(np.unique(t)) > 0.99 * t.size                              # 23-bit draws: few repeats among 8192
    assert (IQ.tau_draw(12345, 8, 2, 64, 64) != t).mean() > 0.99           # the counter moves every draw
    assert (IQ.tau_draw(12346, 7, 2, 64, 64) != t).mean() > 0.99
    assert (t[0] != t[1]).mean() > 0.99                                     # the slots draw independently
    assert abs(float(t.mean()) - 0.5) < 0.02


def _problem(A, N, seed, kappa):
    from oracle import dqn_oracle as O
    rs = np.random.RandomState(seed)
    B = 3
    ws = O.xavier_init(A, seed) + [(rs.uniform(-1, 1, (3136, 64)) * np.sqrt(3.0 / 64)).astype(F32)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.1) * np.abs(w).max()).astype(F32) for w in ws]
    pre = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    act = rs.randint(0, A, B)
    rew = np.array([1, -1, 0])
    term = np.array([False, True, False])
    taus = IQ.tau_draw(seed, 0, 2, B, N)
    return ws, tws, (pre, act, rew, post, term), taus


@pytest.mark.parametrize("kappa", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("N", [1, 2, 8, 64])
@pytest.mark.parametrize("A", [1, 4, 18])
def test_numpy_step_matches_torch_autograd(kappa, N, A):
    """The loss and all six layers' gradients of the numpy step against autograd of sum_b sum_i mean_j rho in float64,
    with the targets T held fixed as the step holds them."""
    torch = pytest.importorskip("torch")
    from oracle import dqn_oracle as O
    ws, tws, mb, taus = _problem(A, N, 100 + N + A, kappa)
    pre, act, rew, post, term = mb
    B = len(act)
    cost, grads, T, _ = IQ.numpy_step([w.copy() for w in ws], [np.zeros_like(w) for w in ws], tws, mb, taus, kappa)
    tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in ws]
    h = torch.from_numpy(pre).double() / 255.0
    for li, (r, s_, k, st) in enumerate(O.CONV_GEOM):
        w = tw[li].reshape(h.shape[1], r, s_, k).permute(3, 0, 1, 2)
        h = torch.relu(torch.nn.functional.conv2d(h, w, stride=st))
    psi = h.flatten(1)
    tau0 = torch.tensor(taus[0], dtype=torch.float64)
    c = torch.cos(torch.pi * torch.arange(64, dtype=torch.float64)[None, :] * tau0[:, None])
    phi = torch.relu(c @ tw[5].T)
    x = psi.repeat_interleave(N, dim=0) * phi
    theta = (torch.relu(x @ tw[3].T) @ tw[4].T).reshape(B, N, A)
    sel = theta[torch.arange(B), :, torch.tensor(act)]                      # (B, N)
    u = torch.tensor(T, dtype=torch.float64)[:, None, :] - sel[:, :, None]
    wgt = torch.abs(tau0.reshape(B, N)[:, :, None] - (u < 0).double())
    if kappa > 0:
        au = u.abs()
        rho = wgt * torch.where(au <= kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa)) / kappa
    else:
        rho = wgt * u.abs()
    loss = rho.mean(dim=2).sum()
    loss.backward()
    assert abs(cost * B - float(loss)) <= 1e-4 * max(abs(float(loss)), 1e-3)
    for layer in range(6):
        ref = tw[layer].grad.numpy()
        err = np.linalg.norm(grads[layer] - ref) / max(np.linalg.norm(ref), 1e-30)
        assert err <= 1e-4, (kappa, N, A, layer, err)


def test_constant_embedding_limit():
    """With phi = 1 (We row 0 = 1, the rest 0) every theta row of a sample is the same, and dWe reduces to its i = 0
    row's form: column i of the Neon (3136, 64) gradient is sum_r c[r][i] dphi[r], column 0 the plain sum of dphi."""
    ws, tws, mb, taus = _problem(4, 8, 5, 1.0)
    we = np.zeros((3136, 64), F32)
    we[:, 0] = 1
    ws[5] = we
    theta, acts = IQ.forward(ws, mb[0], taus[0])
    assert (acts["phi"] == 1).all()
    assert (theta.reshape(3, 8, -1) == theta.reshape(3, 8, -1)[:, :1]).all()
    deltas = np.zeros_like(theta)
    deltas[:, 1] = np.linspace(-1, 1, len(theta)).astype(F32)
    g5 = IQ.backward(ws, acts, deltas)[5]
    d = deltas @ ws[4]
    dphi = ((d * (acts["h4"] > 0)) @ ws[3]) * np.repeat(acts["flat"], 8, axis=0)
    assert np.allclose(g5[:, 0], dphi.sum(axis=0), rtol=1e-4, atol=1e-6)
    assert np.allclose(g5, dphi.T @ acts["c"], rtol=1e-4, atol=1e-6)


def test_restatement_pieces():
    """The device-order pieces: row-order dWe and mod_bwd agree with the vectorised float64 forms, and A = 1 picks
    action 0."""
    rs = np.random.RandomState(1)
    c = IQ.cos_features(IQ.tau_draw(1, 0, 1, 4, 8)[0])
    assert (c[:, 0] == 1).all()
    dphi = rs.randn(32, 40).astype(F32)
    assert np.allclose(IQ.we_grad(c, dphi), c.T.astype(np.float64) @ dphi, rtol=1e-5, atol=1e-5)
    dx, ph, psi = rs.randn(32, 40).astype(F32), np.maximum(rs.randn(32, 40), 0).astype(F32), \
        np.maximum(rs.randn(4, 40), 0).astype(F32)
    dpsi, dph = IQ.mod_bwd(dx, ph, psi, 8)
    ref = (dx * ph).reshape(4, 8, 40).sum(axis=1) * (psi > 0)
    assert np.allclose(dpsi, ref, rtol=1e-5, atol=1e-6)
    assert (dph == np.where(ph > 0, dx * np.repeat(psi, 8, axis=0), 0)).all()
    theta = rs.randn(2, 8, 1).astype(F32)
    _, _, astar, _, _, _ = IQ.head(theta, np.full(8, 0.5, F32), [0], [(0.0, 0.99)], 1.0, 8)
    assert astar[0] == 0


def test_net_create_refuses_before_device_work():
    """num_tau_samples outside 0..64, num_quantile_samples outside 1..64, a second head, a non-finite clip_error or more
    than 4096 expanded rows are EINVAL; dueling and Munchausen are ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.num_tau_samples == 0 and cfg.num_quantile_samples == 32 and cfg.tau_seed == 0
    for fields, exc, match in (({"num_tau_samples": -1}, AssertionError, "num_tau_samples"),
                               ({"num_tau_samples": 65}, AssertionError, "num_tau_samples"),
                               ({"num_quantile_samples": 0}, AssertionError, "num_quantile_samples"),
                               ({"num_quantile_samples": 65}, AssertionError, "num_quantile_samples"),
                               ({"num_atoms": 51}, AssertionError, "one"),
                               ({"num_quantiles": 8}, AssertionError, "one"),
                               ({"clip_error": float("inf")}, AssertionError, "clip_error"),
                               ({"batch_size": 65, "num_tau_samples": 64}, AssertionError, "4096"),
                               ({"batch_size": 129, "num_tau_samples": 1}, AssertionError, "4096"),
                               ({"dueling": 1}, NotImplementedError, "IQN"),
                               ({"munchausen": 1}, NotImplementedError, "IQN")):
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.num_tau_samples = 8
        for k, v in fields.items():
            setattr(cfg, k, v)
        with pytest.raises(exc, match=match):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
