"""CPU checks of tests/qr_oracle.py, the restatement the GPU tests hold the quantile-regression head to: its loss and
quantile gradient against torch autograd of sum_i mean_j rho in float64, a whole-network numpy step against autograd
through the net, the edge cases (a point mass, one action, one quantile), and the creation refusals, which fire ahead
of any device work."""
import ctypes as C

import numpy as np
import pytest

import qr_oracle as QR

F32 = np.float32
EPS = 2.0 ** -24


def _torch_loss(T, th, kappa):
    """sum_i mean_j |tau_i - 1{u_ij < 0}| huber_kappa(u_ij) / kappa (or |u| at kappa = 0), float64, and d/dtheta."""
    torch = pytest.importorskip("torch")
    n = len(th)
    tau = torch.tensor([(2 * i + 1) / (2 * n) for i in range(n)], dtype=torch.float64)
    t = torch.tensor(np.asarray(T, np.float64))
    x = torch.tensor(np.asarray(th, np.float64), requires_grad=True)
    u = t[None, :] - x[:, None]
    w = torch.abs(tau[:, None] - (u < 0).double())
    if kappa > 0:
        au = u.abs()
        hub = torch.where(au <= kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa))
        rho = w * hub / kappa
    else:
        rho = w * u.abs()
    loss = rho.mean(dim=1).sum()
    loss.backward()
    return float(loss.detach()), x.grad.numpy(), rho.detach().numpy()


def _cases(n, kappa, seed):
    rs = np.random.RandomState(seed)
    scale = max(kappa, 0.3) * 2.0
    T = (rs.randn(n) * scale).astype(F32)
    th = (rs.randn(n) * scale + 0.1).astype(F32)
    if n > 2:   # exact ties u = 0 and |u| = kappa: the branch edges of rules 7 and 8
        th[0] = T[1]
        if kappa > 0:
            th[1] = F32(T[2] - F32(kappa))
    return T, th


@pytest.mark.parametrize("kappa", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("n", [1, 2, 51, 200])
def test_loss_and_gradient_match_torch_autograd(kappa, n):
    """The restated row loss and dtheta equal float64 autograd of sum_i mean_j rho within fp32 rounding: each pair term
    takes a few roundings, the j sums N, the i sum N, so the error is below (2N + 8) eps times the sum of |terms|."""
    for seed in range(3):
        T, th = _cases(n, kappa, seed)
        ref_l, ref_g, rho64 = _torch_loss(T, th, kappa)
        l, g = QR.loss_and_grad(T, th, kappa)
        tol_l = (2 * n + 8) * EPS * np.abs(rho64).sum() / n * 4 + 1e-300
        assert abs(float(l) - ref_l) <= tol_l, (seed, float(l), ref_l, tol_l)
        _, c = QR.pair_terms(T, th, kappa)
        tol_g = (n + 8) * EPS * np.abs(c.astype(np.float64)).sum(axis=1) / n * 4 + 1e-300
        assert (np.abs(g.astype(np.float64) - ref_g) <= tol_g).all(), (seed, np.abs(g - ref_g).max())


def test_restatement_is_sensitive_to_its_rules():
    """A swapped weight, a left-out mean over j or an unshifted midpoint each move the result well past the bound."""
    T, th = _cases(51, 1.0, 5)
    l, g = QR.loss_and_grad(T, th, 1.0)
    wlo, whi = QR.taus(51)
    assert wlo[0] == F32(1 / 102) and whi[0] == F32(101 / 102) and (wlo + whi == 1).all()
    ref_l, ref_g, _ = _torch_loss(T, th, 1.0)
    assert abs(float(l) * 51 - ref_l) > 1.0 and np.abs(g * 51 - ref_g).max() > 1e-2


def test_point_mass_has_zero_loss_and_gradient():
    """Every online quantile and every target quantile at one value c: u = 0 everywhere, so the loss and dtheta are 0,
    at any kappa; with a terminal (g = 0) the targets are the return itself."""
    for kappa in (0.0, 1.0):
        for n in (1, 7, 200):
            c = F32(0.75)
            T = QR.targets(0.75, 0.0, np.full(n, 123.0, F32))
            assert (T == c).all()
            l, g = QR.loss_and_grad(T, np.full(n, c, F32), kappa)
            assert l == 0 and (g == 0).all()


def test_one_action_picks_action_zero():
    rs = np.random.RandomState(0)
    theta = rs.randn(3, 5, 1, 9).astype(F32)
    astar, T, _, _ = QR.head(theta, np.zeros(5, np.int64), [(0.5, 0.9)] * 5, 1.0, double=True)
    assert (astar == 0).all()
    for b in range(5):
        assert (T[b] == QR.targets(0.5, 0.9, theta[1, b, 0])).all()


def test_one_quantile_is_median_regression():
    """N = 1: tau = 0.5, both weights 0.5; kappa = 0 gives dtheta = -0.5 sign(T - theta) and loss 0.5 |T - theta|."""
    wlo, whi = QR.taus(1)
    assert wlo[0] == F32(0.5) and whi[0] == F32(0.5)
    for T, th in ((2.0, 1.0), (-1.0, 3.5), (0.25, 0.25)):
        l, g = QR.loss_and_grad(np.array([T], F32), np.array([th], F32), 0.0)
        assert l == F32(0.5) * abs(F32(T) - F32(th))
        assert g[0] == -F32(0.5) * F32(np.sign(T - th))
    # the Q of one quantile is that quantile
    assert QR.q_values(np.array([[3.25]], F32))[0] == F32(3.25)


def test_numpy_step_matches_torch_autograd_of_the_whole_network():
    """The numpy QR step's gradients of all five layers equal torch autograd of sum_b sum_i mean_j rho through the whole
    network (oracle.dqn_torch's forward, in float64), with the targets from the target network held fixed."""
    torch = pytest.importorskip("torch")
    from oracle import dqn_oracle as O
    A, N, B = 3, 5, 4
    rs = np.random.RandomState(2)
    ws = [np.asarray(w, F32) for w in O.xavier_init(A * N, 5)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.1) * np.abs(w).max()).astype(F32) for w in ws]
    pre = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    act = rs.randint(0, A, B)
    rew = np.array([1, -1, 0, 2])
    term = np.array([False, True, False, False])
    w0 = [w.copy() for w in ws]
    for kappa in (1.0, 0.0):
        wk = [w.copy() for w in w0]
        _, grads, T, _ = QR.numpy_step(wk, [np.zeros_like(w) for w in wk], tws, (pre, act, rew, post, term), N, kappa)
        tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in w0]
        h = torch.from_numpy(pre).double() / 255.0
        for li, (r, s_, k, st) in enumerate(O.CONV_GEOM):
            w = tw[li].reshape(h.shape[1], r, s_, k).permute(3, 0, 1, 2)
            h = torch.relu(torch.nn.functional.conv2d(h, w, stride=st))
        theta = (torch.relu(h.flatten(1) @ tw[3].T) @ tw[4].T).reshape(B, A, N)
        sel = theta[torch.arange(B), torch.tensor(act)]
        tau = torch.tensor([(2 * i + 1) / (2 * N) for i in range(N)], dtype=torch.float64)
        u = torch.tensor(T, dtype=torch.float64)[:, None, :] - sel[:, :, None]
        wgt = torch.abs(tau[None, :, None] - (u < 0).double())
        if kappa > 0:
            au = u.abs()
            rho = wgt * torch.where(au <= kappa, 0.5 * u * u, kappa * (au - 0.5 * kappa)) / kappa
        else:
            rho = wgt * u.abs()
        rho.mean(dim=2).sum().backward()
        for layer in range(5):
            ref = tw[layer].grad.numpy()
            err = np.linalg.norm(grads[layer] - ref) / max(np.linalg.norm(ref), 1e-30)
            assert err <= 1e-4, (kappa, layer, err)


def test_net_create_refuses_before_device_work():
    """num_quantiles outside 0..200, together with atoms, or with a non-finite clip_error is EINVAL; with the dueling
    network it is ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.num_quantiles == 0
    for nq, exc, fields in ((-1, AssertionError, {}), (201, AssertionError, {}),
                            (200, AssertionError, {"num_atoms": 51}), (1, AssertionError, {"num_atoms": 2}),
                            (51, AssertionError, {"clip_error": float("inf")}),
                            (51, AssertionError, {"clip_error": float("nan")}),
                            (51, NotImplementedError, {"dueling": 1})):
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.num_quantiles = nq
        for k, v in fields.items():
            setattr(cfg, k, v)
        with pytest.raises(exc, match="quantile"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
