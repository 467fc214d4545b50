"""CPU checks of tests/bootstrap_oracle.py, the restatement the GPU tests hold bootstrapped DQN heads to: the mask hash
against Python-integer test vectors; chi-square tests that the masks are Bernoulli(p) and independent across heads and
ring slots; the head gradient and the 1/K-scaled gradient into the shared network against float64 torch autograd, with
and without importance weights and with Double DQN; the whole network's gradients against autograd; one head at p = 1
as the scalar DQN step; and the creation refusals, which fire ahead of any device work."""
import ctypes as C

import numpy as np
import pytest

import bootstrap_oracle as BOOT

F32 = np.float32
EPS = 2.0 ** -24
M64 = (1 << 64) - 1


def _mix(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def test_masks_match_python_integer_vectors():
    """Rule 1 written out with Python integers, independently of rem_oracle: u = (2 (h >> 9) + 1) / 2^24 from the high
    32 bits h of the hash at the ring slot, m = [u < p] in float64."""
    from simple_dqn_b200.deepqnetwork import bootstrap_seed
    for seed, slot, K, p in ((bootstrap_seed(7), 0, 4, 0.5), (bootstrap_seed(3), 2999, 200, 0.1), (0, 0, 1, 0.9),
                             (M64, 123456789, 17, 0.5), (bootstrap_seed(1), 5, 10, 1.0)):
        base = _mix((seed + 0x9E3779B97F4A7C15 * (slot + 1)) & M64)
        u = [(((_mix(base ^ k) >> 32) >> 9) * 2 + 1) / 2 ** 24 for k in range(K)]
        assert (BOOT.uniforms(seed, slot, K) == np.array(u, F32)).all()
        assert (BOOT.masks(seed, [slot], K, p)[0] == np.array([v < p for v in u], np.uint8)).all()
    assert [int(v * 2 ** 24) for v in BOOT.uniforms(bootstrap_seed(7), 3, 4)] == [
        ((_mix(_mix((bootstrap_seed(7) + 0x9E3779B97F4A7C15 * 4) & M64) ^ k) >> 32) >> 9) * 2 + 1 for k in range(4)]


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_masks_are_bernoulli_and_independent(p):
    """Over 3000 ring slots and 8 heads: the count of ones fits Binomial(p) per head (chi-square), and neighbouring
    heads of one slot and one head of neighbouring slots are independent (2x2 contingency chi-square)."""
    stats = pytest.importorskip("scipy.stats")
    from simple_dqn_b200.deepqnetwork import bootstrap_seed
    K, N = 8, 3000
    m = BOOT.masks(bootstrap_seed(11), range(N), K, p).astype(np.int64)
    for k in range(K):
        ones = int(m[:, k].sum())
        assert stats.chisquare([ones, N - ones], [N * p, N * (1 - p)]).pvalue > 1e-4, (k, ones)
    ones = int(m.sum())
    assert stats.chisquare([ones, N * K - ones], [N * K * p, N * K * (1 - p)]).pvalue > 1e-4

    def independent(x, y):
        t = np.array([[np.sum((x == i) & (y == j)) for j in (0, 1)] for i in (0, 1)])
        return stats.chi2_contingency(t).pvalue > 1e-4

    for k in range(K - 1):
        assert independent(m[:, k], m[:, k + 1]), ("heads", k)
        assert independent(m[:-1, k], m[1:, k]), ("slots", k)


def test_p_one_gives_all_ones():
    assert (BOOT.masks(5, range(500), 200, 1.0) == 1).all()
    u = np.concatenate([BOOT.uniforms(5, i, 200) for i in range(50)])
    assert (u > 0).all() and (u < 1).all()


def _torch_head(theta, h4, w5_block, m, a, y, clip, w=None):
    """float64 autograd of sum_k m_k w huber(theta[a][k] - y_k) (0.5 x^2 when clip = 0) with theta = H4 W5 and the 1/K
    on the shared path only: returns (dtheta (A, K), dH4 (512,))."""
    torch = pytest.importorskip("torch")
    K = len(y)
    h = torch.tensor(np.asarray(h4, np.float64), requires_grad=True)
    hs = h / K + (h - h / K).detach()                  # the value of H4, the gradient scaled by 1/K
    wb = torch.tensor(np.asarray(w5_block, np.float64))   # (512, K) W5's block of the taken action
    th = torch.tensor(np.asarray(theta, np.float64), requires_grad=True)
    ta = hs @ wb                                        # theta[a] as a function of H4, for the gradient only
    d = (th[a] + (ta - ta.detach())) - torch.tensor(np.asarray(y, np.float64))
    ad = d.abs()
    loss = torch.where(ad <= clip, 0.5 * d * d, clip * (ad - 0.5 * clip)) if clip else 0.5 * d * d
    loss = (loss * torch.tensor(np.asarray(m, np.float64))).sum()
    if w is not None:
        loss = loss * float(w)
    loss.backward()
    return th.grad.numpy(), h.grad.numpy()


def _torch_targets(theta_b, ret, double):
    """y_k = R + g theta[1][a*_k][k] in float64 torch, independently of the oracle: a*_k = torch.argmax (the first
    maximum) over the actions of column k of slot 2 with Double DQN, of slot 1 without; theta_b is (3, A, K)."""
    torch = pytest.importorskip("torch")
    th = torch.tensor(np.asarray(theta_b, np.float64))
    astar = torch.argmax(th[2 if double else 1], dim=0)                 # (K,)
    q = th[1].gather(0, astar[None, :])[0]
    R, g = ret
    return (R + g * q).numpy()


@pytest.mark.parametrize("K", [1, 2, 10, 200])
@pytest.mark.parametrize("clip", [0.0, 1.0])
@pytest.mark.parametrize("weighted,double", [(False, False), (True, False), (False, True)])
def test_head_and_shared_gradients_match_torch_autograd(K, clip, weighted, double):
    """dtheta (rule 4) and dZ4 (rule 5: the mean over the heads, into the shared network) equal float64 autograd of
    (1/K) sum_k m_k w huber(theta_k - y_k) with the 1/K applied only to the shared path, within the fp32 roundings of
    y, delta, the clip, the weight and dZ4's K products and sums.  y is formed in float64 torch from its own per-head
    argmax, over slot 2 with Double DQN (the online network on the poststates picks, the target network values), and
    is held fixed."""
    rs = np.random.RandomState(K + 7 * int(weighted) + 3 * int(double))
    A, n = 4, 6
    h4 = np.maximum(rs.randn(n, 512), 0).astype(F32)
    w5 = (rs.randn(512, A * K) * 0.05).astype(F32)           # internal layout [512][A K]
    theta = np.stack([BOOT.logits(h4, w5)] + [(rs.randn(n, A * K) * 2).astype(F32) for _ in range(2)])
    theta = theta.reshape(3, n, A, K)
    acts = rs.randint(0, A, n)
    returns = [(float(rs.randint(-1, 2)), 0.0 if b == 2 else 0.99) for b in range(n)]
    m = BOOT.masks(9, range(100, 100 + n), K, 0.5)
    w = (rs.rand(n) + 0.2).astype(F32) if weighted else None
    q, T, D, cost, err, g = BOOT.head(theta, acts, returns, m, clip, double=double, w=w)
    if double:   # the online network's choice differs from the target network's, so the case is not vacuous
        assert (np.argmax(theta[2], axis=1) != np.argmax(theta[1], axis=1)).any()
    for b in range(n):
        a = int(acts[b])
        y = _torch_targets(theta[:, b], returns[b], double)
        # the oracle's float32 targets are y rounded once (its one-step fma rounds once more than y's product here)
        assert (np.abs(T[b].astype(np.float64) - y) <= 2 * EPS * np.abs(y)).all(), (b, T[b], y)
        ref_th, ref_h = _torch_head(theta[0, b], h4[b], w5[:, a * K:(a + 1) * K], m[b], a, y, clip,
                                    None if w is None else w[b])
        full = np.zeros((A, K), F32)
        full[a] = g[b]
        wt = 1.0 if w is None else float(w[b])
        scale = np.abs(theta[0, b, a]).max() + np.abs(T[b]).max()
        assert (np.abs(full - ref_th) <= 4 * EPS * scale * wt + 1e-300).all(), (b, np.abs(full - ref_th).max())
        assert (ref_th[np.arange(A) != a] == 0).all()
        assert (ref_th[a][m[b] == 0] == 0).all() and (g[b][m[b] == 0] == 0).all()
        dz = BOOT.dz4(h4[b], w5, a, g[b])
        ref_dz = np.where(h4[b] > 0, ref_h, 0.0)
        bound = (K + 4) * EPS * (np.abs(w5[:, a * K:(a + 1) * K]).astype(np.float64) @ np.abs(ref_th[a])) / K
        assert (np.abs(dz - ref_dz) <= bound * 4 + 1e-300).all(), (b, np.abs(dz - ref_dz).max())
    assert np.allclose(err, np.abs(D.astype(np.float64)).mean(axis=1), rtol=(K + 2) * EPS, atol=0)


def _whole_net_autograd(w0, tws, mb, K, m, clip):
    torch = pytest.importorskip("torch")
    from oracle import dqn_oracle as O
    pre, act, rew, post, term = mb
    B = len(act)

    def net(ws, states, shared_scale=False):
        h = torch.from_numpy(states).double() / 255.0
        for li, (r, s_, k, st) in enumerate(O.CONV_GEOM):
            w = ws[li].reshape(h.shape[1], r, s_, k).permute(3, 0, 1, 2)
            h = torch.relu(torch.nn.functional.conv2d(h, w, stride=st))
        h4 = torch.relu(h.flatten(1) @ ws[3].T)
        if shared_scale:
            h4 = h4 / K + (h4 - h4 / K).detach()
        return h4 @ ws[4].T

    tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in w0]
    th = net(tw, pre, True).reshape(B, -1, K)[torch.arange(B), torch.tensor(act)]          # (B, K)
    with torch.no_grad():
        qn = net([torch.tensor(w, dtype=torch.float64) for w in tws], post).reshape(B, -1, K).max(dim=1).values
    r = torch.tensor(np.clip(rew, -1, 1), dtype=torch.float64)[:, None]
    y = r + 0.99 * qn * torch.tensor(~term, dtype=torch.float64)[:, None]
    d = th - y
    ad = d.abs()
    loss = torch.where(ad <= clip, 0.5 * d * d, clip * (ad - 0.5 * clip)) if clip else 0.5 * d * d
    (loss * torch.tensor(m, dtype=torch.float64)).sum().backward()
    return [t.grad.numpy() for t in tw]


@pytest.mark.parametrize("K,clip", [(3, 1.0), (5, 0.0)])
def test_numpy_step_matches_torch_autograd_of_the_whole_network(K, clip):
    """The numpy bootstrapped step's gradients of all five layers equal torch autograd through the whole network
    (float64) of sum_b sum_k m_k huber(theta_k - y_k), with the 1/K on the shared path and y held fixed."""
    from oracle import dqn_oracle as O
    A, B = 3, 4
    rs = np.random.RandomState(2)
    ws = [np.asarray(w, F32) for w in O.xavier_init(A * K, 5)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.1) * np.abs(w).max()).astype(F32) for w in ws]
    mb = (rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8), rs.randint(0, A, B), np.array([1, -1, 0, 2]),
          rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8), np.array([False, True, False, False]))
    m = BOOT.masks(13, range(B), K, 0.5)
    m[0, 0] = 1   # at least one live head, so that every layer gets a gradient
    w0 = [w.copy() for w in ws]
    _, grads, _ = BOOT.numpy_step(ws, [np.zeros_like(w) for w in ws], tws, mb, K, m, clip=clip)
    ref = _whole_net_autograd(w0, tws, mb, K, m, clip)
    for layer in range(5):
        err = np.linalg.norm(grads[layer] - ref[layer]) / max(np.linalg.norm(ref[layer]), 1e-30)
        assert err <= 1e-4, (layer, err)


def test_one_head_at_p_one_is_the_scalar_dqn_step():
    """K = 1, p = 1: the mask is 1 and one bootstrapped step equals the scalar DQN oracle's step within float64 bounds
    (the dot products are summed in other orders, so not bit for bit)."""
    from oracle import dqn_oracle as O
    m = BOOT.masks(3, range(8), 1, 1.0)
    assert (m == 1).all()
    rs = np.random.RandomState(4)
    A, B = 4, 8
    ws = [np.asarray(w, F32) for w in O.xavier_init(A, 9)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    mb = (rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8), rs.randint(0, A, B), rs.randint(-2, 3, B),
          rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8), rs.rand(B) < 0.3)
    orc = O.DQNOracle(A, batch_size=B, weights=[w.copy() for w in ws])
    tws = [w.copy() for w in orc.target_weights]
    rw, rsx = [w.copy() for w in ws], [np.zeros_like(w) for w in ws]
    cost, grads, _ = BOOT.numpy_step(rw, rsx, tws, mb, 1, m)
    ref_cost = orc.train(mb)
    assert abs(cost - float(ref_cost)) <= 1e-5 * abs(float(ref_cost))
    for layer in range(5):
        assert np.linalg.norm(grads[layer] - orc.last["grads"][layer]) <= 1e-5 * np.linalg.norm(orc.last["grads"][layer])
        assert np.linalg.norm(rw[layer] - orc.weights[layer]) <= 1e-5 * np.linalg.norm(orc.weights[layer] - ws[layer])


def test_predict_rule():
    rs = np.random.RandomState(1)
    theta = rs.randn(5, 4, 10).astype(F32)
    for h in range(10):
        assert (BOOT.predict_q(theta, h) == theta[..., h]).all()
    s = np.zeros((5, 4), F32)
    for k in range(10):
        s = (s + theta[..., k]).astype(F32)
    assert (BOOT.predict_q(theta, -1) == (s / F32(10)).astype(F32)).all()


def test_seeds_are_distinct_streams():
    from simple_dqn_b200.deepqnetwork import bootstrap_seed, rem_seed, shift_seed, tau_seed
    for s in (0, 1, 7, 12345):
        assert len({bootstrap_seed(s), rem_seed(s), shift_seed(s), tau_seed(s)}) == 4
        assert bootstrap_seed(s) == bootstrap_seed(s) and 0 <= bootstrap_seed(s) < 1 << 64


def test_net_create_refuses_before_device_work():
    """bootstrap_heads outside 0..200, p outside (0, 1] or not finite, or K beside another head is EINVAL; with the
    dueling network or the Munchausen target it is ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.bootstrap_heads == 0 and cfg.bootstrap_p == 0.5 and cfg.bootstrap_seed == 0
    cases = [(-1, AssertionError, {}), (201, AssertionError, {}),
             (10, AssertionError, {"bootstrap_p": 0.0}), (10, AssertionError, {"bootstrap_p": 1.5}),
             (10, AssertionError, {"bootstrap_p": float("nan")}), (10, AssertionError, {"bootstrap_p": -0.5}),
             (10, AssertionError, {"bootstrap_p": float("inf")}),
             (200, AssertionError, {"num_atoms": 51}), (1, AssertionError, {"num_quantiles": 2}),
             (10, AssertionError, {"num_tau_samples": 8}), (10, AssertionError, {"num_heads": 10}),
             (10, AssertionError, {"num_fractions": 8}),
             (10, NotImplementedError, {"dueling": 1}), (10, NotImplementedError, {"munchausen": 1})]
    for k, exc, fields in cases:
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.bootstrap_heads = k
        for name, v in fields.items():
            setattr(cfg, name, v)
        with pytest.raises(exc, match="bootstrap"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
