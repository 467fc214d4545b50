"""tests/c51_oracle.py against independent computations (CPU): the projection against exact Fraction arithmetic and
against the usual floor/ceil scatter form, mass conservation, the logit gradient against torch autograd of the
cross-entropy, and the support and argument checks of net_create."""
import ctypes as C
import itertools
import math
from fractions import Fraction

import numpy as np
import pytest

import c51_oracle as C51

F32 = np.float32
ATOMS = [2, 3, 51, 64]
SUPPORTS = [(-10.0, 10.0), (-1.0, 3.0), (0.0, 1.0), (-200.0, 0.5)]
GAMMAS = [0.0, 0.5, 0.99, 1.0]


def _cases(atoms, v, seed):
    """(R, g) pairs: n-step returns at N = 1 and 3 with terminal and non-terminal windows, plus returns past both ends."""
    g = np.random.default_rng(seed)
    out = []
    for gamma, n, term in itertools.product(GAMMAS, (1, 3), (False, True)):
        rewards = g.integers(-3, 4, n)
        terminals = np.zeros(n, bool)
        if term:
            terminals[g.integers(0, n)] = True
        out.append(C51.n_step_return(rewards, terminals, gamma, -1, 1))
    span = v[1] - v[0]
    out += [(v[0] - 3 * span, 0.99), (v[1] + 3 * span, 0.99), (v[0], 1.0), (v[1], 1.0), (v[0] - 1e-9, 0.0)]
    return out


def _q(atoms, seed):
    p = np.random.default_rng(seed).random(atoms)
    return (p / p.sum()).astype(F32)


def _exact(R, g, q, atoms, v):
    """The projection in exact rational arithmetic from the same fp64 inputs."""
    vmin, vmax = Fraction(v[0]), Fraction(v[1])
    dz = (vmax - vmin) / (atoms - 1)
    m = [Fraction(0)] * atoms
    for j in range(atoms):
        T = min(max(Fraction(R) + Fraction(g) * (vmin + j * dz), vmin), vmax)
        b = (T - vmin) / dz
        for i in range(atoms):
            m[i] += Fraction(float(q[j])) * max(Fraction(0), 1 - abs(b - i))
    return m


def _scatter(R, g, q, z, v, dz):
    """The usual floor/ceil scatter form, with its l == u case."""
    m = np.zeros(len(z))
    for j in range(len(z)):
        T = min(max(R + g * z[j], v[0]), v[1])
        b = (T - v[0]) / dz
        lo, up = math.floor(b), math.ceil(b)
        lo, up = min(max(lo, 0), len(z) - 1), min(max(up, 0), len(z) - 1)   # b may round a hair past either end
        if lo == up:
            m[lo] += float(q[j])
        else:
            m[lo] += float(q[j]) * (up - b)
            m[up] += float(q[j]) * (b - lo)
    return m


@pytest.mark.parametrize("atoms", ATOMS)
@pytest.mark.parametrize("v", SUPPORTS)
def test_projection_against_exact_and_scatter(atoms, v):
    """Each m_i is within BOUND of the exact projection and of the scatter form; sum(m) = sum(q) within rounding.
    BOUND: the fp64 chain's relative error (a few ulp per term over atoms terms, amplified by 1/dz in b_j) plus the
    final float32 rounding."""
    z, _, dz = C51.support(atoms, *v)
    span = v[1] - v[0]
    for k, (R, g) in enumerate(_cases(atoms, v, atoms)):
        q = _q(atoms, k)
        m = C51.project(R, g, q, z, v[0], v[1], dz)
        ex = _exact(R, g, q, atoms, v)
        sc = _scatter(R, g, q, z, v, dz)
        scale = (abs(R) + abs(g) * max(abs(v[0]), abs(v[1])) + span) / dz
        bound = 2.0 ** -24 + atoms * 8 * scale * 2.0 ** -53
        for i in range(atoms):
            assert abs(float(m[i]) - float(ex[i])) <= bound, (R, g, i)
            assert abs(float(m[i]) - sc[i]) <= bound, (R, g, i)
        assert abs(float(np.sum(m, dtype=np.float64)) - float(np.sum(q, dtype=np.float64))) <= atoms * bound


def test_projection_on_an_atom_and_terminal():
    """A return landing exactly on an atom puts q_j there whole; a terminal (g = 0) puts all mass next to R."""
    z, _, dz = C51.support(51, -10.0, 10.0)
    q = np.zeros(51, F32)
    q[20] = F32(1)
    m = C51.project(2.0, 1.0, q, z, -10.0, 10.0, dz)     # R + z_20 = 2 - 2 = 0 = z_25
    assert m[25] == F32(1) and (np.delete(m, 25) == 0).all()
    q = _q(51, 3)
    m = C51.project(0.0, 0.0, q, z, -10.0, 10.0, dz)
    acc = 0.0
    for v in q:
        acc = acc + float(v)
    assert m[25] == F32(acc) and (np.delete(m, 25) == 0).all()


@pytest.mark.parametrize("atoms", [2, 51, 64])
def test_logit_grad_matches_autograd(atoms):
    torch = pytest.importorskip("torch")
    g = np.random.default_rng(atoms)
    l = (g.standard_normal((8, atoms)) * 5).astype(F32)
    m = g.random((8, atoms)).astype(F32)
    m /= m.sum(axis=1, keepdims=True)
    t = torch.tensor(l, dtype=torch.float64, requires_grad=True)
    loss = torch.nn.functional.cross_entropy(t, torch.tensor(m, dtype=torch.float64), reduction="sum")
    loss.backward()
    p = C51.softmax(l)
    for b in range(8):
        gl = C51.logit_grad(p[b], m[b])
        assert np.allclose(gl, t.grad[b].numpy(), rtol=0, atol=1e-6)
        assert abs(float(C51.loss(m[b], l[b])) -
                   float(torch.nn.functional.cross_entropy(t[b:b + 1].detach(), torch.tensor(m[b:b + 1],
                                                                                              dtype=torch.float64)))) <= 1e-4


def test_fc2_grad_matches_autograd_of_the_head():
    """dW5 of rule 11 equals torch autograd of sum_b CE(logits_b[a_b], m_b) through fc2, for H4 and W5 given."""
    torch = pytest.importorskip("torch")
    g = np.random.default_rng(1)
    A, K, B = 3, 5, 6
    h4 = np.maximum(g.standard_normal((B, 512)), 0).astype(F32)
    w5 = (g.standard_normal((A * K, 512)) * 0.05).astype(F32)
    act = g.integers(0, A, B)
    m = g.random((B, K)).astype(F32)
    m /= m.sum(axis=1, keepdims=True)
    l = C51.logits(h4, w5.T).reshape(B, A, K)
    p = C51.softmax(l)
    gl = np.stack([C51.logit_grad(p[b, act[b]], m[b]) for b in range(B)])
    W = torch.tensor(w5, dtype=torch.float64, requires_grad=True)
    H = torch.tensor(h4, dtype=torch.float64, requires_grad=True)
    L = (H @ W.T).reshape(B, A, K)
    sel = L[torch.arange(B), torch.tensor(act)]
    torch.nn.functional.cross_entropy(sel, torch.tensor(m, dtype=torch.float64), reduction="sum").backward()
    assert np.allclose(C51.fc2_grad(h4, gl, act, A), W.grad.numpy(), rtol=1e-4, atol=1e-5)
    dz4 = np.stack([C51.dz4(h4[b], w5.T, act[b], gl[b]) for b in range(B)])
    assert np.allclose(dz4, H.grad.numpy() * (h4 > 0), rtol=1e-4, atol=1e-5)


def test_net_create_refuses_bad_supports_before_any_device_work():
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    for atoms, lo, hi in ((1, -10.0, 10.0), (65, -10.0, 10.0), (51, 1.0, 1.0), (51, 2.0, 1.0),
                          (51, -float("inf"), 1.0), (51, 0.0, float("nan")), (-1, -10.0, 10.0)):
        cfg = L.NetConfig()
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        assert (cfg.num_atoms, cfg.v_min, cfg.v_max) == (0, -10.0, 10.0)
        cfg.num_atoms, cfg.v_min, cfg.v_max = atoms, lo, hi
        with pytest.raises(AssertionError):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))


def test_numpy_step_matches_torch_autograd_of_the_whole_network():
    """The numpy C51 step's gradients of all five layers equal torch autograd of sum_b CE(logits_b[a_b], m_b) through
    the whole network (oracle.dqn_torch's forward in float64), m from the target network's projected distribution."""
    torch = pytest.importorskip("torch")
    from oracle import dqn_oracle as O
    A, K, B = 3, 11, 4
    rs = np.random.RandomState(2)
    ws = [np.asarray(w, F32) for w in O.xavier_init(A * K, 5)]
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.1) * np.abs(w).max()).astype(F32) for w in ws]
    pre = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (B, 4, 84, 84)).astype(np.uint8)
    act = rs.randint(0, A, B)
    rew = np.array([1, -1, 0, 2])
    term = np.array([False, True, False, False])
    w0 = [w.copy() for w in ws]
    _, grads, m, _ = C51.numpy_step(ws, [np.zeros_like(w) for w in ws], tws, (pre, act, rew, post, term), K, -2.0, 2.0)
    tw = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in w0]
    h = torch.from_numpy(pre).double() / 255.0
    for li, (r, s_, k, st) in enumerate(O.CONV_GEOM):      # oracle.dqn_torch's forward, in float64
        w = tw[li].reshape(h.shape[1], r, s_, k).permute(3, 0, 1, 2)
        h = torch.relu(torch.nn.functional.conv2d(h, w, stride=st))
    logits = (torch.relu(h.flatten(1) @ tw[3].T) @ tw[4].T).reshape(B, A, K)
    sel = logits[torch.arange(B), torch.tensor(act)]
    torch.nn.functional.cross_entropy(sel, torch.tensor(m, dtype=torch.float64), reduction="sum").backward()
    for layer in range(5):
        ref = tw[layer].grad.numpy()
        err = np.linalg.norm(grads[layer] - ref) / max(np.linalg.norm(ref), 1e-30)
        assert err <= 1e-4, (layer, err)
