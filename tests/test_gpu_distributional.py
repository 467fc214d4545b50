"""The distributional value head (C51) on the device against tests/c51_oracle.py, each stage fed the device's own inputs
so that errors do not carry over: H4 against a scalar twin, the logits against the restated fp32 dot products, the
probabilities within CUDA's expf bound of float64, and everything downstream of the probabilities (Q rows, a*, the
projected target, the logit gradient, dZ4, fc2's gradient and its update under every optimizer) bit for bit, on both
engines and both schedules, with Double DQN, prioritized replay and n-step returns.  Also the train paths against each
other, the predict paths, checkpoints, the target sync and the refusals."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import c51_oracle as C51
from helpers import make_args
from oracle import dqn_oracle as O
from oracle.replay_oracle import ReplayOracle, synthetic_ring
from test_gpu_nstep import _mem

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS = 2.0 ** -24


def _L():
    from simple_dqn_b200 import _lib as L
    return L


def _dnet(mode, A=4, atoms=51, v=(-10.0, 10.0), batch=32, hist=4, stream=None, double=False, seed=3, scale=3.0,
          optimizer="rmsprop", target_steps=10000, discount=0.99):
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, history_length=hist, random_seed=seed, double_dqn=double,
                                    distributional=True, num_atoms=atoms, v_min=v[0], v_max=v[1], optimizer=optimizer,
                                    target_steps=target_steps, discount_rate=discount), math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(scale)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [[np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for _ in range(net.num_states)]
                         for w in ws])
    if target_steps:
        net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                        None, which=1)
    return net


def _ring_pair(batch=32, hist=4, stream=None, seed=4, size=3000, terminal_p=0.05, **kw):
    ring = ReplayOracle(size, history_length=hist, batch_size=batch)
    synthetic_ring(ring, seed=seed, block=100, terminal_p=terminal_p)
    mem = _mem(size, hist=hist, batch=batch, stream=stream, **kw)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    return ring, mem


def _gather(ring, idx, n):
    import nstep_oracle as NS
    return NS.gather(ring, np.asarray(idx, np.int64), n)


def _state(net):
    ws, _ = net.get_weights()
    return ws, net.get_states()


def _same_state(a, b):
    (wa, sa), (wb, sb) = _state(a), _state(b)
    for x, y in zip(wa, wb):
        assert (x == y).all()
    for x, y in zip(sa, sb):
        for p, q in zip(x, y):
            assert (p == q).all()


def _check_probs(logits, probs):
    """PROBS within CUDA's documented expf error (2 ulp) of the float64 softmax of the device's logits, with the
    rounding of l - max, of the i-order sum and of the division."""
    l64 = np.asarray(logits, np.float64)
    mx = l64.max(axis=-1, keepdims=True)
    e = np.exp(l64 - mx)
    p64 = e / e.sum(axis=-1, keepdims=True)
    K = l64.shape[-1]
    span = (mx - l64.min(axis=-1, keepdims=True))
    rel_e = 2 * 2.0 ** -23 + span * EPS
    tol = p64 * (2 * rel_e + (K + 2) * EPS) * 1.5 + 2.0 ** -140
    assert (np.abs(np.asarray(probs, np.float64) - p64) <= tol).all()


def _loss_bound(m, l_row):
    """|row cost - float64 cross-entropy| bound: expf 2 ulp and logf 1 ulp (CUDA), one rounding per operation."""
    l = np.asarray(l_row, np.float64)
    m = np.asarray(m, np.float64)
    mx = l.max()
    ls = np.log(np.exp(l - mx).sum())
    logp = l - mx - ls
    K = len(l)
    rel_s = 2 * 2.0 ** -23 + (mx - l.min()) * EPS + K * EPS
    abs_ls = rel_s * 1.01 + 2 * 2.0 ** -23 * abs(ls)
    term = EPS * np.abs(l - mx) + abs_ls + EPS * (np.abs(l - mx) + abs(ls)) + EPS * np.abs(logp)
    exact = -(m * logp).sum()
    return exact, 2 * ((m * term).sum() + (K + 2) * EPS * np.abs(m * logp).sum()) + 1e-30


def _optimize(optimizer, w, states, g, batch, t=1):
    """oracle.dqn_oracle's update of one layer, in place on copies."""
    w = w.copy()
    states = [s.copy() for s in states]
    if optimizer == "rmsprop":
        O.rmsprop_update([w], [states[0]], [g], batch)
    elif optimizer == "adam":
        O.adam_update([w], [states[:2]], [g], batch, t)
    else:
        O.adadelta_update([w], [states[:3]], [g], batch)
    return w, states


def _slot_h4(net, weights, states):
    """H4 of `weights` on `states` from a scalar twin's predict: an independent source for slots 1 and 2."""
    from simple_dqn_b200 import DeepQNetwork
    twin = DeepQNetwork(net.num_actions, make_args(batch_size=net.batch_size, history_length=net.history_length),
                        math_mode=net.math_mode)
    tw = twin.get_weights(with_states=False)
    twin.set_weights(list(weights[:4]) + [tw[4]])
    twin.predict(states)
    return twin.last_activations()[3]


def _check_train_step(net, before, actions, rewards, terminals, post, discount=0.99, lo=-1, hi=1, w=None, td=False,
                      separate=True):
    """Every stage of the last train step fed the device's own inputs.  before = (weights, states) ahead of the step;
    rewards / terminals are (batch, N) windows, post the poststates the target slots read; separate: the target
    network is not the online one."""
    A, K, b = net.num_actions, net.num_atoms, len(actions)
    z, zf, dz = C51.support(K, net.v_min, net.v_max)
    assert (net.support == z).all()
    probs, logits = net.last_distributions(), net.last_logits()
    two = net.double_dqn and separate
    nets = 3 if two else 2
    _check_probs(logits[:nets], probs[:nets])
    # logits: the restated fp32 dot products of the device's H4 and W5 (slot 0, online weights before the step)
    h4 = net.last_activations()[3]
    w5 = before[0][4]
    assert (logits[0].reshape(b, A * K) == C51.logits(h4, w5.T)).all()
    # slot 1: the target network on the poststates; slot 2 (Double DQN): the online network on the poststates
    tws = net.get_weights(which=1, with_states=False) if separate else before[0]
    h4t = _slot_h4(net, tws, post)
    assert (logits[1].reshape(b, A * K) == C51.logits(h4t, tws[4].T)).all()
    if two:
        h4o = _slot_h4(net, before[0], post)
        assert (logits[2].reshape(b, A * K) == C51.logits(h4o, w5.T)).all()
    preq, postq = net.last_q()
    assert (preq == C51.q_values(probs[0], zf)).all()
    assert (postq == C51.q_values(probs[1], zf)).all()
    if two:
        assert (net.last_online_postq() == C51.q_values(probs[2], zf)).all()
    rewards, terminals = np.asarray(rewards), np.asarray(terminals)
    returns = [C51.n_step_return(rewards[i], terminals[i], discount, lo, hi) for i in range(b)]
    _, m, gl = C51.head(probs, actions, returns, z, net.v_min, net.v_max, dz, double=two, w=w)
    assert (net.last_target_distribution() == m).all()
    assert (net.last_logit_grads() == gl).all()
    dz4 = net.last_dz()[3]
    for i in range(b):
        assert (dz4[i] == C51.dz4(h4[i], w5.T, actions[i], gl[i])).all(), i
    if net.math_mode == "tcgen05":          # the fp16 planes the tensor-core fc1 dgrad and wgrad read
        hi16, lo16 = net.last_dz4_planes()
        ehi, elo = C51.fp16_planes(dz4)
        assert (hi16.view(np.uint16) == ehi.view(np.uint16)).all() and (lo16.view(np.uint16) == elo.view(np.uint16)).all()
    rc = net.last_row_costs()
    tde = net.last_td_errors() if td else None
    for i in range(b):
        exact, tol = _loss_bound(m[i], logits[0, i, actions[i]])
        wi = 1.0 if w is None else float(w[i])
        assert abs(float(rc[i]) - wi * exact) <= wi * tol + abs(wi * exact) * EPS, (i, rc[i], exact, tol)
        if td:
            assert abs(float(tde[i]) - exact) <= tol, i
            assert rc[i] == F32(F32(w[i]) * tde[i])
    tot = F32(0)
    for c in rc:
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(b))
    g = C51.fc2_grad(h4, gl, actions, A)
    assert (net.get_grads()[4] == g).all()
    w_new, s_new = _optimize(net.optimizer, w5, before[1][4], g, b)
    ws, ss = _state(net)
    assert (ws[4] == w_new).all()
    for k in range(net.num_states):
        assert (ss[4][k] == s_new[k]).all(), k
    return m, gl


# ---------------------------------------------------------------------------------------------------- forward
FORWARD = [  # (mode, batch, A, atoms, v, scale)
    ("tcgen05", 1, 1, 2, (-10.0, 10.0), 3.0), ("fp32", 33, 4, 51, (-1.0, 3.0), 3.0),
    ("tcgen05", 257, 18, 64, (0.0, 1.0), 3.0), ("fp32", 1, 32, 64, (-200.0, 0.5), 3.0),
    ("tcgen05", 33, 32, 51, (-10.0, 10.0), 300.0), ("tcgen05", 4096, 4, 51, (-10.0, 10.0), 3.0),
    ("fp32", 257, 4, 2, (-1.0, 3.0), 300.0),
]


@pytest.mark.parametrize("mode,batch,A,atoms,v,scale", FORWARD)
def test_predict_forward_stages(mode, batch, A, atoms, v, scale):
    """H4 equals a scalar twin's with the same conv and fc1 weights; the logits equal the restated fp32 dot products
    of the device's H4 and W5; the probabilities are within the expf bound; Q equals the restated expectation."""
    from simple_dqn_b200 import DeepQNetwork
    net = _dnet(mode, A=A, atoms=atoms, v=v, batch=batch, scale=scale)
    twin = DeepQNetwork(A, make_args(batch_size=batch, random_seed=5), math_mode=mode)
    ws, _ = net.get_weights()
    tws = twin.get_weights(with_states=False)
    twin.set_weights(ws[:4] + [tws[4]])
    states = np.random.RandomState(batch + A).randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    q = net.predict(states)
    twin.predict(states)
    h4 = net.last_activations()[3]
    assert (h4 == twin.last_activations()[3]).all()
    logits = net.last_logits()[0]
    assert (logits.reshape(batch, A * atoms) == C51.logits(h4, ws[4].T)).all()
    probs = net.last_distributions()[0]
    _check_probs(logits, probs)
    assert np.isfinite(probs).all()
    assert (q == C51.q_values(probs, net.support.astype(F32))).all()


# ---------------------------------------------------------------------------------------------------- train step
ENGINES = [("tcgen05", "branches"), ("fp32", "branches"), ("tcgen05", "serial"), ("fp32", "serial")]
STEP = [  # (batch, A, atoms, v, n, discount, hist)
    (33, 4, 51, (-10.0, 10.0), 1, 0.99, 4), (1, 1, 2, (-1.0, 3.0), 3, 1.0, 1), (257, 18, 64, (0.0, 1.0), 1, 0.0, 4),
    (33, 32, 64, (-200.0, 0.5), 16, 0.99, 16), (33, 4, 2, (-10.0, 10.0), 3, 0.99, 1),
]


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("batch,A,atoms,v,n,discount,hist", STEP)
def test_train_step_stages(mode, sched, double, per, batch, A, atoms, v, n, discount, hist):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream() if sched == "branches" else None
    ring, mem = _ring_pair(batch=batch, hist=hist, stream=stream, prioritized_replay=per, beta0=0.4, terminal_p=0.1)
    ring.actions[:] = np.random.RandomState(batch).randint(0, A, len(ring.actions))
    from test_gpu_prioritized import _upload
    _upload(mem, _L().PTR_ACTIONS, ring.actions)
    mem.set_n_step(n)
    net = _dnet(mode, A=A, atoms=atoms, v=v, batch=batch, hist=hist, stream=stream, double=double, discount=discount)
    before = _state(net)
    idx = np.array(random.Random(batch * 7 + n).sample(range(hist, 3000 - n + 1), batch), np.int32)
    mem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    mb = _gather(ring, idx, n)
    _check_train_step(net, before, mb[1].astype(np.int64), mb[2], mb[4], mb[3], discount=discount,
                      w=mem.last_weights if per else None, td=per)
    if per:   # the tree's leaves after the priority update: (|loss| + eps)^alpha, CUDA's pow within 2 ulp
        pr = mem.priorities
        exp = np.array([(abs(float(d)) + mem.eps) ** mem.alpha for d in net.last_td_errors()])
        assert (np.abs(pr[idx] - exp) <= 2 * np.spacing(exp)).all()


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("optimizer", ["rmsprop", "adam", "adadelta"])
@pytest.mark.parametrize("target_steps", [10000, 0])
def test_optimizers_and_target_steps_zero(mode, optimizer, target_steps):
    """A host-minibatch step under every optimizer (Adam's step scalar comes from the new head), with and without a
    separate target network, Double DQN on; discount 0.99 and terminals mixed."""
    from helpers import random_minibatch
    net = _dnet(mode, A=4, atoms=51, batch=33, optimizer=optimizer, target_steps=target_steps, double=True)
    before = _state(net)
    pre, act, rew, post, term = random_minibatch(33, 4, 5)
    net.train((pre, act, rew, post, term))
    _check_train_step(net, before, act.astype(np.int64), rew[:, None], term[:, None], post,
                      separate=target_steps != 0)


BOUND_CASES = {"default": (-1, 1), "half": (-0.5, 0.5), "inverted": (1, -1), "infinite": (-float("inf"), float("inf")),
               "huge": (-3e9, 3e9)}


@pytest.mark.parametrize("bounds", sorted(BOUND_CASES))
@pytest.mark.parametrize("terminals", ["none", "all", "mixed"])
def test_reward_bounds_and_terminals(bounds, terminals):
    """Rewards out to the int64 extremes under every reward-bound case: returns land past both ends of the support."""
    from simple_dqn_b200 import DeepQNetwork
    lo, hi = BOUND_CASES[bounds]
    net = DeepQNetwork(4, make_args(batch_size=33, min_reward=lo, max_reward=hi, distributional=True, num_atoms=51,
                                    v_min=-10.0, v_max=10.0), math_mode="tcgen05")
    before = _state(net)
    g = np.random.default_rng(8)
    big = np.array([2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 63 - 1, -(2 ** 63 - 1)] + list(range(-7, 8)), np.int64)
    rs = np.random.RandomState(2)
    pre = rs.randint(0, 256, (33, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (33, 4, 84, 84)).astype(np.uint8)
    act = rs.randint(0, 4, 33).astype(np.uint8)
    rew = g.choice(big, 33)
    term = {"none": np.zeros(33, bool), "all": np.ones(33, bool), "mixed": rs.rand(33) < 0.5}[terminals]
    net.train((pre, act, rew, post, term))
    _check_train_step(net, before, act.astype(np.int64), rew[:, None], term[:, None], post, lo=lo, hi=hi)


# ---------------------------------------------------------------------------------------------------- paths
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_ring_step_equals_host_minibatch_step(mode):
    """Two steps from the ring (the captured step graph) equal the same steps from host tuples, bit for bit."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    net = _dnet(mode, stream=stream)
    twin = _dnet(mode, stream=Stream())
    for step in range(2):
        idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
        mem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, idx, 1)
        twin.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
        assert (net.last_costs(1) == twin.last_costs(1)).all()
        assert (net.last_target_distribution() == twin.last_target_distribution()).all()
        _same_state(net, twin)


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_train_fused_equals_sample_then_train_sampled(mode):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream, tstream = Stream(), Stream()
    _, mem = _ring_pair(stream=stream)
    _, tmem = _ring_pair(stream=tstream)
    net = _dnet(mode, stream=stream, double=True)
    twin = _dnet(mode, stream=tstream, double=True)
    random.seed(4)
    mem.seed_device_rng(random)
    for _ in range(3):
        key = mem.read_device_rng()
        _L().call("b200dqn_replay_set_rng", tmem._h, _L().np_ptr(key), tmem._stream)
        tmem._rng_on_device = True
        net.train_fused(mem, 1)
        tmem.sample()
        twin.train(DeviceMinibatch(tmem, sampled=True))
        assert (net.last_costs(1) == twin.last_costs(1)).all()
        _same_state(net, twin)


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_agent_loop_in_lock_step(mode):
    """getMinibatch / train with the process-global `random`: the host stream stays equal to the oracle's, and each
    step's target distribution equals the restatement."""
    from oracle.mt19937 import MT19937
    import nstep_oracle as NS
    from simple_dqn_b200 import Stream
    stream = Stream()
    ring = ReplayOracle(1500, batch_size=32)
    synthetic_ring(ring, seed=2, block=100, terminal_p=0.03)
    mem = _mem(1500, rng="python", stream=stream)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    net = _dnet(mode, stream=stream)
    random.seed(13)
    for _ in range(3):
        before = _state(net)
        rng = MT19937.from_python(random)
        idx, _ = NS.sample_indexes(ring, rng, 1)
        mb = mem.getMinibatch()
        net.train(mb)
        assert list(random.getstate()[1]) == rng.state625()
        g = _gather(ring, idx, 1)
        _check_train_step(net, before, g[1].astype(np.int64), g[2], g[4], g[3])


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_predict_paths_agree(mode):
    """Host predict, predict_device and the captured fast path agree bit for bit on the live row; padding rows come
    back as exact zeros."""
    from simple_dqn_b200 import StateBuffer, Stream
    stream = Stream()
    net = _dnet(mode, stream=stream)
    sb = StateBuffer(make_args(), stream=stream)
    rs = np.random.RandomState(1)
    for _ in range(4):
        sb.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    ds = sb.getStateMinibatch()
    fast = net.predict(ds)
    fast2 = net.predict(ds)
    host = net.predict(np.asarray(ds))
    L = _L()
    qp = net.device_view(L.NET_PTR_Q_ONLINE, (32, 4)).ptr
    L.call("b200dqn_net_predict_device", net._h, C.c_void_p(ds.device_ptr()), 1, C.c_void_p(qp), net._stream)
    dev = net._read_f32(L.NET_PTR_Q_ONLINE, (32, 4))
    assert (fast[0] == host[0]).all() and (fast2 == fast).all() and (dev[0] == host[0]).all()
    assert (fast[1:] == 0).all() and (dev[1:] == 0).all()
    assert (host[1:] != 0).any()                       # zero frames give mean(z) under this head, not 0


# ---------------------------------------------------------------------------------------------------- state
@pytest.mark.parametrize("layout", ["neon-1.3.0", "pre-1.0"])
def test_checkpoints_and_target_sync(layout, tmp_path):
    from simple_dqn_b200 import DeepQNetwork
    net = _dnet("tcgen05", optimizer="adam")
    net.train(__import__("helpers").random_minibatch(32, 4, 3))
    path = os.path.join(str(tmp_path), "c51.pkl")
    net.save_weights(path, layout=layout)
    other = _dnet("tcgen05", optimizer="adam", seed=9)
    other.load_weights(path)
    _same_state(net, other)
    scalar = DeepQNetwork(4, make_args(), math_mode="tcgen05")
    with pytest.raises(AssertionError):
        scalar.load_weights(path)
    spath = os.path.join(str(tmp_path), "scalar.pkl")
    scalar.save_weights(spath, layout=layout)
    with pytest.raises(AssertionError):
        other.load_weights(spath)
    net.update_target_network()
    assert (net.get_weights(which=1, with_states=False)[4] == net.get_weights(with_states=False)[4]).all()
    L = _L()
    for k in range(net.num_states):
        a, b = np.empty((4 * 51, 512), F32), np.empty((4 * 51, 512), F32)
        L.call("b200dqn_net_get_state", net._h, 0, 4, k, L.np_ptr(a), None)
        L.call("b200dqn_net_get_state", net._h, 1, 4, k, L.np_ptr(b), None)
        assert (a == b).all()


def test_refusals_and_launch_counts():
    from simple_dqn_b200 import DeepQNetwork, Stream
    for kw in ({"num_atoms": 1}, {"num_atoms": 65}, {"v_min": 1.0, "v_max": 1.0}, {"v_min": 2.0, "v_max": 1.0},
               {"v_min": -float("inf")}, {"v_max": float("nan")}):
        args = dict(distributional=True, num_atoms=51, v_min=-10.0, v_max=10.0)
        args.update(kw)
        with pytest.raises(AssertionError):
            DeepQNetwork(4, make_args(**args), math_mode="tcgen05")
    net = _dnet("tcgen05")
    with pytest.raises(NotImplementedError, match="distributional"):
        net.comm_init(bytes(128), 0, 2)
    with pytest.raises(AssertionError):
        net.last_deltas()
    scalar = DeepQNetwork(4, make_args(), math_mode="tcgen05")
    with pytest.raises(AssertionError):
        scalar.last_logits()
    for mode in ("tcgen05", "fp32"):
        stream = Stream()
        _, mem = _ring_pair(stream=stream)
        random.seed(1)
        mem.seed_device_rng(random)
        counts = []
        for dist in (False, True):
            n = _dnet(mode, stream=stream) if dist else DeepQNetwork(4, make_args(), math_mode=mode, stream=stream)
            n.train_fused(mem, 1)
            counts.append(n.launches_per_step())
        assert counts[1] == counts[0] + (1 if mode == "tcgen05" else 2), counts


# ---------------------------------------------------------------------------------------------------- rest of the net
@pytest.mark.parametrize("batch", [1, 33, 257])
@pytest.mark.parametrize("sched", ["serial", "branches"])
def test_backbone_kernels_within_float64_bounds(batch, sched):
    """With dZ4 from the distributional head, every tensor-core kernel of the step stays inside the float64 bound its
    hi/lo scheme promises (tests/test_gpu_kernels.py's yardstick), forward and backward."""
    import kernel_ref as K
    from helpers import random_minibatch
    from simple_dqn_b200 import Stream
    from test_gpu_kernels import _chain, _check
    net = _dnet("tcgen05", batch=batch, stream=Stream() if sched == "branches" else None, double=True)
    net.keep_grads(True)
    ws = net.get_weights(with_states=False)
    mb = random_minibatch(batch, 4, 7)
    net.train(mb)
    pre = mb[0]
    h1, h2, h3, h4 = net.last_activations()
    dz1, dz2, dz3, dz4 = net.last_dz()
    grads = net.get_grads()
    c = lambda k: _chain("tcgen05", k, batch, 4)
    fc1_dgrad = lambda a, b: K.fc_dgrad(a, b).reshape(len(a), 64, 7, 7)
    r = {}
    r.update(_check("conv1_fwd", "tcgen05", K.conv_fwd(0), K.states_f64(pre), ws[0], h1, c("conv1_fwd"), post=K.relu,
                    a_exact=True))
    r.update(_check("conv2_fwd", "tcgen05", K.conv_fwd(1), h1, ws[1], h2, c("conv2_fwd"), post=K.relu))
    r.update(_check("conv3_fwd", "tcgen05", K.conv_fwd(2), h2, ws[2], h3, c("conv3_fwd"), post=K.relu))
    r.update(_check("fc1_fwd", "tcgen05", K.fc_fwd, h3, ws[3], h4, c("fc1_fwd"), post=K.relu))
    r.update(_check("fc1_dgrad", "tcgen05", fc1_dgrad, dz4, ws[3], dz3, c("fc1_dgrad"), mask=h3 > 0))
    r.update(_check("conv3_dgrad", "tcgen05", K.conv_dgrad(2), dz3, ws[2], dz2, c("conv3_dgrad"), mask=h2 > 0))
    r.update(_check("conv2_dgrad", "tcgen05", K.conv_dgrad(1), dz2, ws[1], dz1, c("conv2_dgrad"), mask=h1 > 0))
    r.update(_check("fc1_wgrad", "tcgen05", K.fc_wgrad, h3, dz4, grads[3], c("fc1_wgrad")))
    r.update(_check("conv3_wgrad", "tcgen05", K.conv_wgrad(2), h2, dz3, grads[2], c("conv3_wgrad")))
    r.update(_check("conv2_wgrad", "tcgen05", K.conv_wgrad(1), h1, dz2, grads[1], c("conv2_wgrad")))
    r.update(_check("conv1_wgrad", "tcgen05", K.conv_wgrad(0), K.states_f64(pre), dz1, grads[0], c("conv1_wgrad"),
                    a_exact=True))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, bad


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_fused_trajectory_against_a_numpy_c51_step(mode):
    """Five fused steps against tests/c51_oracle.numpy_step (oracle.dqn_oracle's forward, backward and RMSProp with
    the distributional head) on the same minibatches: cost within 1e-3, every layer's update within rel-L2 2e-2."""
    from helpers import rel_l2
    from simple_dqn_b200 import Stream
    from test_gpu_prioritized import _dev
    stream = Stream()
    ring, mem = _ring_pair(stream=stream, terminal_p=0.05)
    net = _dnet(mode, stream=stream)
    ws, ss = _state(net)
    ows, oss = [w.copy() for w in ws], [s[0].copy() for s in ss]
    tws = net.get_weights(which=1, with_states=False)
    w0 = [w.copy() for w in ws]
    random.seed(9)
    mem.seed_device_rng(random)
    for _ in range(5):
        net.train_fused(mem, 1)
        idx = _dev(mem, _L().PTR_INDEXES, np.int32, 32).astype(np.int64)
        mb = _gather(ring, idx, 1)
        ref, _, _, _ = C51.numpy_step(ows, oss, tws, (mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]), 51, -10.0, 10.0)
        cost = float(net.last_costs(1)[0])
        assert abs(cost - ref) <= 1e-3 * abs(ref), (cost, ref)
    got = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(got[l] - w0[l], ows[l] - w0[l]) <= 2e-2, l
