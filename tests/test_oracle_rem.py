"""CPU checks of tests/rem_oracle.py, the restatement the GPU tests hold the random ensemble mixture (REM) head to: the
mixture generator against Python-integer test vectors, its positivity, normalisation and freshness; the head gradient
and the whole network's gradients against torch autograd of sum_b huber(Q_alpha - y) in float64, with and without
importance weights; one head as the scalar DQN step; the Xavier draw; and the creation refusals, which fire ahead of any
device work."""
import ctypes as C

import numpy as np
import pytest

import rem_oracle as REM

F32 = np.float32
EPS = 2.0 ** -24
M64 = (1 << 64) - 1


def _mix(x):
    x ^= x >> 30
    x = (x * 0xBF58476D1CE4E5B9) & M64
    x ^= x >> 27
    x = (x * 0x94D049BB133111EB) & M64
    return x ^ (x >> 31)


def test_mixture_matches_python_integer_vectors():
    """Rule 1 written out with Python integers and fractions, independently of iqn_oracle: u_k = (2m + 1) / 2^24 from
    the top 23 bits of the hash, alpha_k the fp32 rounding of the fp64 quotient."""
    from simple_dqn_b200.deepqnetwork import rem_seed
    for seed, ctr, K in ((rem_seed(7), 0, 4), (rem_seed(3), 5, 200), (0, 0, 1), (M64, 123456789, 17)):
        base = _mix((seed + 0x9E3779B97F4A7C15 * (ctr + 1)) & M64)
        u = [((_mix(base ^ k) >> 32) >> 9) * 2 + 1 for k in range(K)]
        assert (REM.draws(seed, ctr, K) == np.array([v / 2 ** 24 for v in u], F32)).all()
        S = 0.0
        for v in u:
            S += v / 2 ** 24
        assert (REM.alpha(seed, ctr, K) == np.array([F32((v / 2 ** 24) / S) for v in u], F32)).all()
    # a pinned vector, so that a change of the hash shows even if both restatements move together
    assert [int(v * 2 ** 24) for v in REM.draws(rem_seed(7), 0, 4)] == [
        ((_mix(_mix((rem_seed(7) + 0x9E3779B97F4A7C15) & M64) ^ k) >> 32) >> 9) * 2 + 1 for k in range(4)]


@pytest.mark.parametrize("K", [1, 2, 10, 200])
def test_mixture_is_positive_normalised_and_fresh(K):
    """alpha > 0, sum within K fp32 roundings of 1; K = 1 gives exactly 1.0; successive counters draw afresh, and the
    draws look uniform (mean of u near 1/2)."""
    seen = set()
    us = []
    for ctr in range(40):
        al = REM.alpha(99, ctr, K)
        assert (al > 0).all()
        assert abs(float(np.sum(al.astype(np.float64))) - 1.0) <= K * EPS
        if K == 1:
            assert al[0] == F32(1.0)
        else:
            key = al.tobytes()
            assert key not in seen
            seen.add(key)
        us.extend(REM.draws(99, ctr, K))
    us = np.array(us, np.float64)
    assert (us > 0).all() and (us < 1).all()
    assert abs(us.mean() - 0.5) <= 5 * np.sqrt(1 / 12 / len(us))


def _torch_head(theta, al, a, y, clip, w=None):
    """d/dtheta of w * huber_clip(Q_alpha[a] - y) in float64 (0.5 x^2 when clip = 0), theta (A, K)."""
    torch = pytest.importorskip("torch")
    th = torch.tensor(np.asarray(theta, np.float64), requires_grad=True)
    q = th @ torch.tensor(np.asarray(al, np.float64))
    d = q[a] - float(y)
    if clip:
        ad = d.abs()
        loss = torch.where(ad <= clip, 0.5 * d * d, clip * (ad - 0.5 * clip))
    else:
        loss = 0.5 * d * d
    if w is not None:
        loss = loss * float(w)
    loss.backward()
    return th.grad.numpy()


@pytest.mark.parametrize("K", [1, 2, 10, 200])
@pytest.mark.parametrize("clip", [0.0, 1.0])
@pytest.mark.parametrize("weighted", [False, True])
def test_head_gradient_matches_torch_autograd(K, clip, weighted):
    """dtheta (rule 6, at the taken action, 0 elsewhere) equals float64 autograd of w huber(Q_alpha - y) with y held
    fixed, within the fp32 roundings of Q_alpha (K products and sums), delta, the clip, the weight and the product."""
    rs = np.random.RandomState(K)
    A, n = 4, 6
    theta = (rs.randn(3, n, A, K) * 2).astype(F32)
    al = REM.alpha(5, K, K)
    acts = rs.randint(0, A, n)
    returns = [(float(rs.randint(-1, 2)), 0.0 if b == 2 else 0.99) for b in range(n)]
    w = (rs.rand(n) + 0.2).astype(F32) if weighted else None
    q, T, D, cost, g = REM.head(theta, al, acts, returns, clip, w=w)
    for b in range(n):
        ref = _torch_head(theta[0, b], al, acts[b], T[b], clip, None if w is None else w[b])
        full = np.zeros((A, K), F32)
        full[acts[b]] = g[b]
        scale = np.abs(theta[0, b, acts[b]].astype(np.float64) * al).sum() + abs(float(T[b]))
        tol = (K + 6) * EPS * scale * np.abs(al).max() * (1 if w is None else float(w[b])) * 4 + 1e-300
        assert (np.abs(full - ref) <= tol).all(), (b, np.abs(full - ref).max(), tol)
        assert (ref[np.arange(A) != acts[b]] == 0).all()


def _whole_net_autograd(w0, tws, mb, K, al, clip):
    torch = pytest.importorskip("torch")
    from oracle import dqn_oracle as O
    pre, act, rew, post, term = mb
    B = len(act)

    def net(ws, states):
        h = torch.from_numpy(states).double() / 255.0
        for li, (r, s_, k, st) in enumerate(O.CONV_GEOM):
            w = ws[li].reshape(h.shape[1], r, s_, k).permute(3, 0, 1, 2)
            h = torch.relu(torch.nn.functional.conv2d(h, w, stride=st))
        return torch.relu(h.flatten(1) @ ws[3].T) @ ws[4].T

    alt = torch.tensor(np.asarray(al, np.float64))
    tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in w0]
    q = (net(tw, pre).reshape(B, -1, K) @ alt)[torch.arange(B), torch.tensor(act)]
    with torch.no_grad():
        qn = (net([torch.tensor(w, dtype=torch.float64) for w in tws], post).reshape(B, -1, K) @ alt).max(dim=1).values
    r = torch.tensor(np.clip(rew, -1, 1), dtype=torch.float64)
    y = r + 0.99 * qn * torch.tensor(~term, dtype=torch.float64)
    d = q - y
    ad = d.abs()
    loss = torch.where(ad <= clip, 0.5 * d * d, clip * (ad - 0.5 * clip)) if clip else 0.5 * d * d
    loss.sum().backward()
    return [t.grad.numpy() for t in tw]


@pytest.mark.parametrize("K,clip", [(3, 1.0), (5, 0.0)])
def test_numpy_step_matches_torch_autograd_of_the_whole_network(K, clip):
    """The numpy REM step's gradients of all five layers equal torch autograd of sum_b huber(Q_alpha - y) through the
    whole network (float64), with y from the target network held fixed."""
    from oracle import dqn_oracle as O
    A, B = 3, 4
    rs = np.random.RandomState(2)
    ws = [np.asarray(w, F32) for w in O.xavier_init(A * K, 5)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.1) * np.abs(w).max()).astype(F32) for w in ws]
    mb = (rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8), rs.randint(0, A, B), np.array([1, -1, 0, 2]),
          rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8), np.array([False, True, False, False]))
    al = REM.alpha(11, 0, K)
    w0 = [w.copy() for w in ws]
    _, grads, _ = REM.numpy_step(ws, [np.zeros_like(w) for w in ws], tws, mb, K, al, clip=clip)
    ref = _whole_net_autograd(w0, tws, mb, K, al, clip)
    for layer in range(5):
        err = np.linalg.norm(grads[layer] - ref[layer]) / max(np.linalg.norm(ref[layer]), 1e-30)
        assert err <= 1e-4, (layer, err)


def test_one_head_is_the_scalar_dqn_step():
    """K = 1: alpha is exactly 1.0, Q_alpha is theta, and one REM step equals the scalar DQN oracle's step within
    float64 bounds (the dot products are summed in other orders, so not bit for bit)."""
    from oracle import dqn_oracle as O
    assert REM.alpha(3, 0, 1)[0] == F32(1.0)
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
    cost, grads, _ = REM.numpy_step(rw, rsx, tws, mb, 1, np.ones(1, F32))
    ref_cost = orc.train(mb)
    assert abs(cost - float(ref_cost)) <= 1e-5 * abs(float(ref_cost))
    for layer in range(5):
        assert np.linalg.norm(grads[layer] - orc.last["grads"][layer]) <= 1e-5 * np.linalg.norm(orc.last["grads"][layer])
        assert np.linalg.norm(rw[layer] - orc.weights[layer]) <= 1e-5 * np.linalg.norm(orc.weights[layer] - ws[layer])


def test_xavier_shapes_and_draw_order():
    """A REM net's fc2 has Neon shape (A K, 512); every layer is drawn from one RandomState in layer order, so the first
    four are the scalar net's draws and fc2 continues the stream with fan_in 512."""
    from oracle import dqn_oracle as O
    ws = O.xavier_init(4 * 200, 3)
    assert [w.shape for w in ws] == [(256, 32), (512, 64), (576, 64), (512, 3136), (800, 512)]
    base = O.xavier_init(4, 3)
    for l in range(4):
        assert (ws[l] == base[l]).all()
    rng = np.random.RandomState(3)
    for shp in [(256, 32), (512, 64), (576, 64), (512, 3136)]:
        rng.uniform(-1, 1, shp)
    s = np.sqrt(3.0 / 512)
    assert (ws[4] == rng.uniform(-s, s, (800, 512)).astype(F32)).all()


def test_seeds_are_distinct_streams():
    from simple_dqn_b200.deepqnetwork import rem_seed, shift_seed, tau_seed
    for s in (0, 1, 7, 12345):
        assert len({rem_seed(s), shift_seed(s), tau_seed(s)}) == 3
        assert rem_seed(s) == rem_seed(s) and 0 <= rem_seed(s) < 1 << 64


def test_net_create_refuses_before_device_work():
    """num_heads outside 0..200, or with num_atoms, num_quantiles or num_tau_samples, is EINVAL; with the dueling
    network or the Munchausen target it is ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.num_heads == 0 and cfg.rem_seed == 0
    for k, exc, fields in ((-1, AssertionError, {}), (201, AssertionError, {}),
                           (200, AssertionError, {"num_atoms": 51}), (1, AssertionError, {"num_quantiles": 2}),
                           (10, AssertionError, {"num_tau_samples": 8}),
                           (10, NotImplementedError, {"dueling": 1}), (10, NotImplementedError, {"munchausen": 1})):
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.num_heads = k
        for name, v in fields.items():
            setattr(cfg, name, v)
        with pytest.raises(exc, match="num_heads|REM"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
