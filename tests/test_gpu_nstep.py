"""n-step returns on the device ring (b200dqn_replay_set_n_step) against tests/nstep_oracle.py: the draw, the window
the first conv layer reads, the head's n-step target on both engines (vanilla and Double DQN, uniform and
prioritized rings), two identities that need no restatement, the prioritized tree's mask, graph staleness, a
trajectory against the numpy oracle, the agent loop and the refusals."""
import ctypes as C
import random
import types

import numpy as np
import pytest

import nstep_oracle as NS
import per_oracle as P
from helpers import make_args, rel_l2
from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring
from test_gpu_prioritized import _dev, _frames, _net, _state, _upload

pytestmark = pytest.mark.gpu

F32 = np.float32


def _L():
    from simple_dqn_b200 import _lib as L
    return L


def _mem(size, hist=4, batch=32, rng="device", stream=None, **kw):
    from simple_dqn_b200 import ReplayMemory
    return ReplayMemory(size, make_args(history_length=hist, batch_size=batch, **kw), rng=rng, stream=stream)


def _same_state(a, b):
    (wa, sa), (wb, sb) = _state(a), _state(b)
    for x, y in zip(wa, wb):
        assert (x == y).all()
    for x, y in zip(sa, sb):
        for p, q in zip(x, y):
            assert (p == q).all()
    for x, y in zip(a.get_weights(which=1, with_states=False), b.get_weights(which=1, with_states=False)):
        assert (x == y).all()


# ---------------------------------------------------------------------------------------------------- sampler
SAMPLER = [  # (size, hist, n, batch, count, current)
    (50, 4, 3, 32, 50, 20), (50, 1, 2, 1, 50, 0), (50, 16, 16, 257, 50, 37),
    (5000, 4, 3, 4096, 5000, 1234), (5000, 16, 5, 257, 3000, 3000), (70000, 1, 16, 4096, 70000, 69999),
    (1 << 20, 4, 3, 32, 1 << 20, 777), (1 << 20, 16, 16, 4096, 1 << 20, 5),
    # draw widths 1 and 2 (count - H - N + 1), the write pointer just outside and inside the window edges
    (60, 4, 3, 8, 7, 0), (60, 4, 3, 8, 7, 7), (60, 4, 3, 8, 8, 8), (60, 4, 3, 8, 8, 1), (60, 1, 16, 8, 18, 18),
]


@pytest.mark.parametrize("size,hist,n,batch,count,current", SAMPLER)
def test_sampler_equals_cpython(size, hist, n, batch, count, current):
    """Every index, the words consumed and the MT19937 state after each of three draws equal CPython's randint(H,
    count - N) filtered by the n-step window test and the terminal test; N = 1 on the same ring gives the old
    sampler's draw (the reference's)."""
    mem = _mem(size, hist=hist, batch=batch, rng="python")
    g = np.random.default_rng(size + n)
    term = (g.random(size) < (0.0 if count - hist - n < 2 else 0.02)).astype(np.uint8)
    _upload(mem, _L().PTR_TERMINALS, term)
    mem.set_cursor(count, current)
    ring = types.SimpleNamespace(history_length=hist, terminals=term.astype(bool), count=count, current=current,
                                 batch_size=batch)
    for nn in (n, 1):
        mem.set_n_step(nn)
        random.seed(size * 7 + nn)
        for _ in range(3):
            rng = MT19937.from_python(random)
            idx, words = NS.sample_indexes(ring, rng, nn)
            mem.sample()
            assert (_dev(mem, _L().PTR_INDEXES, np.int32, batch) == idx).all()
            assert mem.last_words_consumed == words
            assert list(random.getstate()[1]) == rng.state625()


def test_sampler_edges_of_the_write_pointer():
    """Draw width 2 (indexes H and H + 1): the write pointer at i - H and i + N leaves i drawable, at i - H + 1 and
    i + N - 1 it does not; every draw is also CPython's."""
    hist, n = 4, 3
    mem = _mem(60, hist=hist, batch=16, rng="python")
    mem.set_n_step(n)
    count = hist + n + 1
    for current, drawable in ((0, {4, 5}), (1, {5}), (2, set()), (hist + n, {4}), (hist + n + 1, {4, 5})):
        ring = types.SimpleNamespace(history_length=hist, terminals=np.zeros(60, bool), count=count, current=current,
                                     batch_size=16)
        assert {i for i in (4, 5) if NS.accept(ring, i, n)} == drawable
        if not drawable:
            continue                                    # the reference's loop would never end
        mem.set_cursor(count, current)
        random.seed(current)
        rng = MT19937.from_python(random)
        idx, words = NS.sample_indexes(ring, rng, n)
        mem.sample()
        got = _dev(mem, _L().PTR_INDEXES, np.int32, 16)
        assert (got == idx).all() and set(got.tolist()) <= drawable
        assert mem.last_words_consumed == words and list(random.getstate()[1]) == rng.state625()


# ---------------------------------------------------------------------------------------------------- head
ENGINES = [("tcgen05", "branches"), ("fp32", "branches"), ("tcgen05", "serial")]
SHAPES = [(2, 4, 33), (3, 1, 257), (16, 16, 1), (3, 4, 257), (16, 4, 33), (2, 16, 1)]   # (N, H, batch)


def _ring_pair(batch=32, hist=4, stream=None, seed=4, size=3000, terminal_p=0.05, **kw):
    ring = ReplayOracle(size, history_length=hist, batch_size=batch)
    synthetic_ring(ring, seed=seed, block=100, terminal_p=terminal_p)
    mem = _mem(size, hist=hist, batch=batch, stream=stream, **kw)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    return ring, mem


def _check_head(net, mem, idx, n, mb, double, per, discount=0.99, lo=-1, hi=1):
    preq, postq = net.last_q()
    w = mem.last_weights if per else None
    d, rc, td = NS.head_restated(preq, postq, mb[1], mb[2], mb[4], discount, lo, hi, 1.0, w=w,
                                 online_postq=net.last_online_postq() if double else None)
    assert (net.last_deltas() == d).all()
    assert (net.last_row_costs() == rc).all()
    if per:
        assert (net.last_td_errors() == td).all()
    tot = F32(0)
    for c in rc:
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(len(idx)))


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("per", [False, True])
@pytest.mark.parametrize("n,hist,batch", SHAPES)
def test_head_and_poststates(mode, sched, double, per, n, hist, batch):
    """The head's deltas, row costs, TD errors and cost equal the restatement fed the device's own Q rows; the target
    network's Q (and the online network's on the poststates) equal a twin's host-minibatch step on staged
    getState(i - 1) / getState(i + N - 1), bit for bit."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream() if sched == "branches" else None
    ring, mem = _ring_pair(batch=batch, hist=hist, stream=stream, prioritized_replay=per, beta0=0.5)
    mem.set_n_step(n)
    net = _net(mode, batch=batch, hist=hist, stream=stream, double=double)
    twin = _net(mode, batch=batch, hist=hist, stream=stream, double=double)
    idx = np.array(random.Random(n * 100 + batch).sample(range(hist, 3000 - n + 1), batch), np.int32)
    idx[0] = 3000 - n                     # the last slot whose window fits the ring
    mem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    mb = NS.gather(ring, idx.astype(np.int64), n)
    _check_head(net, mem, idx, n, mb, double, per)
    twin.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
    assert (net.last_q()[1] == twin.last_q()[1]).all()
    assert (net.last_q()[0] == twin.last_q()[0]).all()
    if double:
        assert (net.last_online_postq() == twin.last_online_postq()).all()


BOUND_CASES = {"default": (-1, 1), "half": (-0.5, 0.5), "inverted": (1, -1), "infinite": (-float("inf"), float("inf")),
               "huge": (-3e9, 3e9)}


@pytest.mark.parametrize("bounds", sorted(BOUND_CASES))
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("per", [False, True])
def test_head_at_reward_bounds(bounds, mode, per):
    """Rewards out to the int64 extremes, clipped at float, crossed and infinite bounds, N = 3, discount 0.5."""
    from simple_dqn_b200 import DeepQNetwork, DeviceMinibatch, Stream
    lo, hi = BOUND_CASES[bounds]
    stream = Stream()
    ring, mem = _ring_pair(batch=33, stream=stream, prioritized_replay=per)
    g = np.random.default_rng(8)
    big = np.array([2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 63 - 1, -(2 ** 63 - 1)] + list(range(-7, 8)), np.int64)
    ring.rewards[:] = g.choice(big, 3000)
    _upload(mem, _L().PTR_REWARDS, ring.rewards)
    mem.set_n_step(3)
    net = DeepQNetwork(4, make_args(batch_size=33, min_reward=lo, max_reward=hi, discount_rate=0.5), math_mode=mode,
                       stream=stream)
    idx = np.array(random.Random(3).sample(range(4, 2998), 33), np.int32)
    mem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    _check_head(net, mem, idx, 3, NS.gather(ring, idx.astype(np.int64), 3), False, per, 0.5, lo, hi)


# ---------------------------------------------------------------------------------------------------- identities
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("n", [3, 16])
@pytest.mark.parametrize("identity", ["discount0", "terminal"])
def test_identities_with_the_one_step_step(mode, n, identity):
    """discount_rate = 0: the n-step step is the one-step step on the same indexes.  A sample whose own terminal is
    set has the one-step target at every N.  Deltas, cost and every weight and state plane, bit for bit."""
    from simple_dqn_b200 import DeepQNetwork, DeviceMinibatch, Stream
    out = []
    for nn in (1, n):
        stream = Stream()
        ring, mem = _ring_pair(stream=stream, terminal_p=0.0 if identity == "terminal" else 0.05)
        idx = np.array(random.Random(5).sample(range(200, 2800, 2), 32), np.int32)
        if identity == "terminal":
            t = np.zeros(3000, np.uint8)
            t[idx] = 1
            _upload(mem, _L().PTR_TERMINALS, t)
        mem.set_n_step(nn)
        net = _net(mode, stream=stream)
        if identity == "discount0":
            ref = net
            net = DeepQNetwork(4, make_args(discount_rate=0.0, random_seed=3), math_mode=mode, stream=stream)
            net.set_weights(*_state(ref))
            net.set_weights(ref.get_weights(which=1, with_states=False), None, which=1)
        for step in range(2):
            mem.set_indexes(np.roll(idx, step))
            net.train(DeviceMinibatch(mem, sampled=True))
        out.append((net, net.last_costs(2), net.last_deltas()))
    (a, ca, da), (b, cb, db) = out
    assert (ca == cb).all() and (da == db).all()
    _same_state(a, b)


# ---------------------------------------------------------------------------------------------------- prioritized tree
def _check_mask(mem, n):
    L = _L()
    sz = mem.size
    nl, off = P.layout(sz)
    prio = _dev(mem, L.PTR_PRIORITIES, np.float64, sz)
    sums = P.split_flat(_dev(mem, L.PTR_SUM_TREE, np.float64, off[-1]), sz)
    mins = P.split_flat(_dev(mem, L.PTR_MIN_TREE, np.float64, off[-1] - off[1]), sz, minimum=True)
    count, current = mem._cursor()
    leaves = np.where(NS.valid_mask(mem.terminals, count, current, mem.history_length, n), prio, 0.0)
    assert (sums[0] == leaves).all()
    rs, rm = P.build(sums[0])
    for l in range(1, len(rs)):
        assert (sums[l] == rs[l]).all() and (mins[l - 1] == rm[l]).all()


@pytest.mark.parametrize("n", [1, 3, 16])
@pytest.mark.parametrize("hist", [1, 4])
def test_prioritized_tree_masks_the_window(n, hist):
    """Every leaf and node after single adds across the write pointer and the wrap, add_batch, set_cursor, the switch
    of n_step and a priority update: leaf i is its priority exactly when the n-step draw may take i."""
    from simple_dqn_b200 import DeepQNetwork, DeviceMinibatch
    mem = _mem(80, hist=hist, batch=8, prioritized_replay=True, alpha=0.7)
    mem.set_n_step(n)
    a, r, s, t = _frames(300, n + hist, terminal_p=0.1)
    for i in range(29):
        mem.add(a[i], r[i], s[i], t[i])
        if i % 3 == 0:
            _check_mask(mem, n)
    mem.add_batch(a[29:50], r[29:50], s[29:50], t[29:50])
    _check_mask(mem, n)
    for i in range(50, 190):                               # wraps the ring
        mem.add(a[i], r[i], s[i], t[i])
        if i % 7 == 0:
            _check_mask(mem, n)
    _check_mask(mem, n)
    for count, current in ((80, 7), (80, 79), (40, 40), (80, 0)):
        mem.set_cursor(count, current)
        _check_mask(mem, n)
    mem.set_n_step(1 if n > 1 else 2)
    _check_mask(mem, mem.n_step)
    mem.set_n_step(n)
    _check_mask(mem, n)
    net = DeepQNetwork(4, make_args(batch_size=8, history_length=hist), math_mode="tcgen05")
    mem.set_indexes(np.array([20, 30, 40, 50, 33, 21, 22, 23], np.int32))
    net.train(DeviceMinibatch(mem, sampled=True))
    _check_mask(mem, n)
    for i in range(190, 213):
        mem.add(a[i], r[i], s[i], t[i])
    _check_mask(mem, n)


# ---------------------------------------------------------------------------------------------------- staleness
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("fused", [False, True])
def test_switching_n_step_rebuilds_the_step_graphs(mode, fused):
    """One net trained at N = 1, then 3, then 1 on one ring equals, after every step, a twin on a twin ring that
    trained only at that step's setting (fresh graphs), bit for bit."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    net = _net(mode, stream=stream)
    random.seed(4)
    mem.seed_device_rng(random)
    for step, n in enumerate((1, 3, 1)):
        tstream = Stream()
        _, tmem = _ring_pair(stream=tstream)
        twin = _net(mode, stream=tstream)
        twin.set_weights(*_state(net))
        twin.set_weights(net.get_weights(which=1, with_states=False), None, which=1)
        mem.set_n_step(n)
        tmem.set_n_step(n)
        if fused:
            key = mem.read_device_rng()
            _L().call("b200dqn_replay_set_rng", tmem._h, _L().np_ptr(key), tmem._stream)
            tmem._rng_on_device = True
            net.train_fused(mem, 1)
            twin.train_fused(tmem, 1)
        else:
            idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
            for m, nt in ((mem, net), (tmem, twin)):
                m.set_indexes(idx)
                nt.train(DeviceMinibatch(m, sampled=True))
        assert (net.last_costs(1) == twin.last_costs(1)).all(), step
        assert (net.last_deltas() == twin.last_deltas()).all(), step
        _same_state(net, twin)


# ---------------------------------------------------------------------------------------------------- trajectory
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_fused_trajectory_against_the_numpy_oracle(mode):
    """Five fused N = 3 steps against oracle.dqn_oracle with the n-step target on the same minibatches: cost within
    1e-3, the weight updates within rel-L2 2e-2."""
    from simple_dqn_b200 import Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream, terminal_p=0.05)
    mem.set_n_step(3)
    net = _net(mode, stream=stream)
    ws, ss = _state(net)
    orc = O.DQNOracle(4, batch_size=32, weights=ws, states=[s[0] for s in ss])
    for t, w in zip(orc.target_weights, net.get_weights(which=1, with_states=False)):
        t[...] = w
    w0 = [w.copy() for w in ws]
    random.seed(9)
    mem.seed_device_rng(random)
    for _ in range(5):
        net.train_fused(mem, 1)
        idx = _dev(mem, _L().PTR_INDEXES, np.int32, 32).astype(np.int64)
        ref = NS.train_step(orc, NS.gather(ring, idx, 3))
        cost = net.last_costs(1)[0]
        assert abs(cost - ref) <= 1e-3 * abs(ref)
    got = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(got[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l


# ---------------------------------------------------------------------------------------------------- agent loop
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_agent_loop_in_lock_step(mode):
    """getMinibatch / train at N = 3 with the process-global `random`: a DeviceMinibatch every time, the host stream
    equal to the oracle's after every draw, the statistics materialisation gives the (batch, N) windows and
    getState(index + N - 1), and the materialised minibatch still trains from the ring."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    ring = ReplayOracle(1500, batch_size=32)
    mem = _mem(1500, rng="python", stream=stream, n_step=3)
    assert mem.n_step == 3
    net = _net(mode, stream=stream)
    a, r, s, t = _frames(900, 11, terminal_p=0.03)
    for i in range(600):
        ring.add(a[i], r[i], s[i], t[i])
    mem.add_batch(a[:600], r[:600], s[:600], t[:600])
    random.seed(13)
    pos = 600
    for it in range(6):
        for i in range(pos, pos + 5):
            ring.add(a[i], r[i], s[i], t[i])
            mem.add(a[i], r[i], s[i], t[i])
        pos += 5
        random.random()
        rng = MT19937.from_python(random)
        idx, _ = NS.sample_indexes(ring, rng, 3)
        mb = mem.getMinibatch()
        assert isinstance(mb, DeviceMinibatch)
        if it % 2 == 0:
            pre, act, rew, post, term = mb                   # statistics.py:85 looks at it: the draw happens here
            assert (mem.last_indexes == idx).all()
            exp = NS.gather(ring, idx, 3)
            assert (pre == exp[0]).all() and (post == exp[3]).all() and (act == exp[1]).all()
            assert rew.shape == (32, 3) and (rew == exp[2]).all() and term.dtype == np.bool_ and (term == exp[4]).all()
            net.train(mb)
        else:
            net.train(mb)
        assert (_dev(mem, _L().PTR_INDEXES, np.int32, 32) == idx).all()
        assert list(random.getstate()[1]) == rng.state625()
        mb = NS.gather(ring, idx, 3)
        preq, postq = net.last_q()
        d, _, _ = NS.head_restated(preq, postq, mb[1], mb[2], mb[4])
        assert (net.last_deltas() == d).all()


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals():
    from simple_dqn_b200 import DeepQNetwork, Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    with pytest.raises(AssertionError):
        mem.set_n_step(0)
    with pytest.raises(AssertionError):
        mem.set_n_step(3000 - 4 + 1)
    mem.set_n_step(3000 - 4)                                  # hist + n = size: one index fits
    mem.set_n_step(3)
    with pytest.raises(AssertionError):
        mem.set_indexes(np.full(32, 2998, np.int32))          # the window would run off the ring
    small = _mem(100, rng="python", n_step=5)
    for i in range(8):
        small.add(0, 0, np.zeros((84, 84), np.uint8), False)
    with pytest.raises(AssertionError):
        small.getMinibatch()                                  # count 8 < H + N = 9
    small.add(0, 0, np.zeros((84, 84), np.uint8), False)
    small.getMinibatch()
    net = DeepQNetwork(4, make_args(), math_mode="tcgen05", stream=stream)
    random.seed(1)
    mem.seed_device_rng(random)
    net.train_fused(mem, 1)
    with pytest.raises(NotImplementedError, match="n-step"):
        net.comm_init(bytes(128), 0, 2)
    p, b = C.c_void_p(), C.c_size_t()
    _L().call("b200dqn_replay_device_ptr", mem._h, _L().PTR_MB_REWARDS, C.byref(p), C.byref(b))
    assert b.value == 32 * 3 * 8
