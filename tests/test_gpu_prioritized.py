"""Prioritized experience replay on the device (b200dqn_replay_set_prioritized, csrc/per.cu) against the oracle of
tests/per_oracle.py: the trees after writes and after priority updates, the draw and its weights, the weighted train
step on both engines, the agent loop, the refusals and the off state."""
import ctypes as C
import random

import numpy as np
import pytest

import per_oracle as P
from helpers import make_args
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring

pytestmark = pytest.mark.gpu

F32 = np.float32


def _L():
    from simple_dqn_b200 import _lib as L
    return L


def _dev(mem, which, dtype, n):
    return _L().download(mem.device, mem.device_view(which, dtype, (n,)).ptr, (n,), dtype, mem._stream)


def _upload(mem, which, arr):
    L = _L()
    view = mem.device_view(which, arr.dtype, arr.shape)
    L.call("b200dqn_copy_to_device", mem.device, C.c_void_p(view.ptr), L.np_ptr(np.ascontiguousarray(arr)),
           arr.nbytes, mem._stream)


def device_tree(mem):
    """(stored priorities, sum levels, min levels 1.., terminals, count, current) as the device holds them."""
    L = _L()
    n, off = P.layout(mem.size)
    prio = _dev(mem, L.PTR_PRIORITIES, np.float64, mem.size)
    sums = P.split_flat(_dev(mem, L.PTR_SUM_TREE, np.float64, off[-1]), mem.size)
    mins = P.split_flat(_dev(mem, L.PTR_MIN_TREE, np.float64, off[-1] - off[1]), mem.size, minimum=True)
    count, current = mem._cursor()
    return prio, sums, mins, mem.terminals, count, current


def check_tree(mem, expect_prio=None):
    """Leaves = rule 1 on the device's own ring and priorities, every internal node = the oracle's, bit for bit."""
    prio, sums, mins, term, count, current = device_tree(mem)
    if expect_prio is not None:
        assert (prio == expect_prio).all()
    leaves = np.where(P.valid_mask(term, count, current, mem.history_length), prio, 0.0)
    assert (sums[0] == leaves).all()
    rs, rm = P.build(sums[0])
    for l in range(1, len(rs)):
        assert (sums[l] == rs[l]).all(), l
        assert (mins[l - 1] == rm[l]).all(), l
    return prio, sums, mins, count


def _frames(n, seed, terminal_p=0.05):
    g = np.random.default_rng(seed)
    return (g.integers(0, 4, n).astype(np.uint8), g.integers(-1, 2, n).astype(np.int64),
            g.integers(0, 256, (n, 84, 84), dtype=np.uint8), g.random(n) < terminal_p)


def _mem(size, hist=4, batch=32, rng="device", stream=None, **kw):
    from simple_dqn_b200 import ReplayMemory
    return ReplayMemory(size, make_args(history_length=hist, batch_size=batch, **kw), rng=rng, stream=stream)


# ---------------------------------------------------------------------------------------------------- writes
@pytest.mark.parametrize("hist", [1, 4, 16])
def test_tree_after_writes(hist):
    mem = _mem(50, hist=hist, batch=8, prioritized_replay=True)
    assert mem.prioritized
    ones = np.ones(50)
    check_tree(mem, ones)                                  # empty ring: every leaf 0
    a, r, s, t = _frames(130, hist, terminal_p=0.15)
    for i in range(23):                                    # single adds through the deferred bank
        mem.add(a[i], r[i], s[i], t[i])
    check_tree(mem, ones)
    mem.add_batch(a[23:40], r[23:40], s[23:40], t[23:40])
    check_tree(mem, ones)
    for i in range(40, 130):                               # wraps the ring
        mem.add(a[i], r[i], s[i], t[i])
    assert mem.count == 50
    check_tree(mem, ones)
    for count, current in ((50, 7), (50, 49), (30, 30), (50, 0)):
        mem.set_cursor(count, current)
        check_tree(mem, ones)


def test_writes_take_max_priority():
    """After a train step raised max_priority, new slots get max_priority^alpha; every node follows."""
    from simple_dqn_b200 import DeepQNetwork, DeviceMinibatch, Stream
    stream = Stream()
    mem = _mem(200, batch=8, stream=stream, prioritized_replay=True, alpha=0.7)
    a, r, s, t = _frames(260, 1)
    mem.add_batch(a[:200], r[:200], s[:200], t[:200])
    net = DeepQNetwork(4, make_args(batch_size=8), math_mode="tcgen05", stream=stream)
    mem.set_indexes(np.array([20, 30, 40, 50, 60, 70, 80, 90], np.int32))
    net.train(DeviceMinibatch(mem, sampled=True))
    maxp = mem.max_priority
    td = net.last_td_errors().astype(np.float64)
    assert maxp == max(1.0, float(np.max(np.abs(td) + 1e-6)))
    before = mem.priorities
    for i in range(200, 213):
        mem.add(a[i], r[i], s[i], t[i])
    prio, *_ = check_tree(mem)
    fresh = np.arange(200, 213) % 200
    np.testing.assert_array_max_ulp(prio[fresh], np.full(13, maxp ** 0.7), maxulp=2)
    keep = np.setdiff1d(np.arange(200), fresh)
    assert (prio[keep] == before[keep]).all()


# ---------------------------------------------------------------------------------------------------- draws
DRAWS = [  # (ring size, history, batch, beta0)
    (50, 4, 8, 0.4), (50, 1, 1, 1.0), (5000, 16, 32, 0.4), (5000, 4, 40, 0.0), (100000, 4, 256, 0.4),
    (1 << 20, 4, 32, 0.4), (1 << 20, 16, 4096, 1.0), (70000, 1, 4096, 0.0)]


@pytest.mark.parametrize("size,hist,batch,beta0", DRAWS)
def test_draw_equals_oracle(size, hist, batch, beta0):
    """Indexes bit for bit on the device's tree, weights within 2 ulp, 2 * batch words, the host `random` in
    lock-step, beta annealed over three draws (beta_steps = 2)."""
    mem = _mem(size, hist=hist, batch=batch, rng="python")
    g = np.random.default_rng(size + batch)
    term = (g.random(size) < 0.03).astype(np.uint8)
    _upload(mem, _L().PTR_TERMINALS, term)
    mem.set_prioritized(True, alpha=0.6, beta0=beta0, beta_steps=2)
    _upload(mem, _L().PTR_PRIORITIES, g.random(size) ** 4 + 1e-3)   # stored priorities spanning 4 decades
    mem.set_cursor(size, int(g.integers(0, size)))                  # rebuilds every leaf and node
    random.seed(size)
    for k in range(3):
        _, sums, mins, count = check_tree(mem)
        rng = MT19937.from_python(random)
        idx, w = P.draw(sums, mins, rng, batch, count, k, beta0, 2)
        mem.sample()
        got = _dev(mem, _L().PTR_INDEXES, np.int32, batch)
        assert (got == idx).all()
        np.testing.assert_array_max_ulp(mem.last_weights, w, maxulp=2)
        if beta0 == 0.0 and k == 0:
            assert (mem.last_weights == F32(1)).all()
        assert mem.last_words_consumed == 2 * batch
        assert list(random.getstate()[1]) == rng.state625()


def test_draw_from_a_ring_with_no_drawable_slot_is_an_error():
    mem = _mem(100, batch=8, rng="python", prioritized_replay=True)
    _upload(mem, _L().PTR_TERMINALS, np.ones(100, np.uint8))
    mem.set_cursor(100, 3)
    with pytest.raises(_L().B200DQNError, match="no slot"):
        mem.sample()
    mem.set_prioritized(True)   # clears the sticky error; the ring is still undrawable
    with pytest.raises(_L().B200DQNError):
        mem.sample()


# ---------------------------------------------------------------------------------------------------- train step
def _ring_pair(batch=32, hist=4, stream=None, seed=4, **kw):
    ring = ReplayOracle(3000, history_length=hist, batch_size=batch)
    synthetic_ring(ring, seed=seed, block=100, terminal_p=0.02)
    mem = _mem(3000, hist=hist, batch=batch, stream=stream, **kw)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    return ring, mem


def _net(mode, batch=32, hist=4, stream=None, double=False, seed=3):
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(4, make_args(batch_size=batch, history_length=hist, random_seed=seed, double_dqn=double),
                       math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for w in ws])
    net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                    None, which=1)
    return net


def _state(net):
    ws, _ = net.get_weights()
    return ws, net.get_states()


ENGINES = [("tcgen05", "branches"), ("tcgen05", "serial"), ("fp32", "branches")]


def _stream(sched):
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("alpha", [0.0, 0.6, 1.0])
def test_train_step_head_and_priority_update(mode, sched, double, alpha):
    """The weighted head bit for bit from the device's own Q rows; priorities within 2 ulp of numpy's pow of the
    device's TD errors (repeated slot: the last occurrence wins); every internal node exact over the device leaves."""
    from simple_dqn_b200 import DeviceMinibatch
    stream = _stream(sched)
    ring, mem = _ring_pair(stream=stream, prioritized_replay=True, alpha=alpha, beta0=0.5, beta_steps=10)
    net = _net(mode, stream=stream, double=double)
    pool = random.Random(1).sample(range(500, 2900), 48)
    mem.set_indexes(np.array(pool[:32], np.int32))       # a first step gives 32 slots their own priorities
    net.train(DeviceMinibatch(mem, sampled=True))
    maxp1 = mem.max_priority
    idx = np.array(pool[16:46] + [0, 0], np.int32)
    idx[30], idx[31] = idx[3], idx[7]                     # entries 3 and 7 appear twice
    mem.set_indexes(idx)
    w = mem.last_weights
    prio0, sums0, mins0, count = check_tree(mem)
    ref_w = np.array([P.weight(prio0[i], sums0[-1][0], mins0[-1][0], float(count), 0.5) for i in idx], F32)
    np.testing.assert_array_max_ulp(w, ref_w, maxulp=2)
    net.train(DeviceMinibatch(mem, sampled=True))
    preq, postq = net.last_q()
    mb = ring.gather(idx.astype(np.int64))
    d, rc, td = P.head_restated(preq, postq, mb[1], mb[2], mb[4], w,
                                online_postq=net.last_online_postq() if double else None)
    assert (net.last_deltas() == d).all()
    assert (net.last_td_errors() == td).all()
    tot = F32(0)
    for c in rc:                                          # k_cost_finish: row order, fp32
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(32))
    if alpha > 0:
        assert len(np.unique(w)) > 1
    per = P.PEROracle(ring, alpha=alpha)
    per.prio = prio0.copy()
    per.update(idx, net.last_td_errors())
    prio, *_ = check_tree(mem)
    np.testing.assert_array_max_ulp(prio, per.prio, maxulp=2)
    assert mem.max_priority == max(maxp1, float(np.max(np.abs(td.astype(np.float64)) + 1e-6)))


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("double", [False, True])
def test_beta_zero_step_equals_uniform_step(mode, sched, double):
    """At beta = 0 every weight is 1.0f, so the prioritized step is the uniform step on the same indexes, bit for bit:
    cost, deltas, weights and every optimizer state plane."""
    from simple_dqn_b200 import DeviceMinibatch
    stream = _stream(sched)
    ring, mem = _ring_pair(stream=stream)
    nets = [_net(mode, stream=stream, double=double) for _ in range(2)]
    idx = np.array(random.Random(2).sample(range(100, 2900), 32), np.int32)
    for net, on in zip(nets, (True, False)):
        mem.set_prioritized(on, beta0=0.0, beta_steps=1e9)
        for step in range(2):
            mem.set_indexes(np.roll(idx, step))
            if on:
                assert (mem.last_weights == F32(1)).all()
            net.train(DeviceMinibatch(mem, sampled=True))
    a, b = nets
    assert (a.last_costs(2) == b.last_costs(2)).all()
    assert (a.last_deltas() == b.last_deltas()).all()
    (wa, sa), (wb, sb) = _state(a), _state(b)
    for x, y in zip(wa, wb):
        assert (x == y).all()
    for x, y in zip(sa, sb):
        for p, q in zip(x, y):
            assert (p == q).all()


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("batch", [32, 256])
def test_fused_step_equals_sample_and_train_sampled(mode, batch):
    """train_fused on a prioritized ring (draw, weighted step, priority update in one graph, beta annealing over the
    steps) equals sample() + train_sampled, bit for bit, over five steps."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    out = []
    for fused in (True, False):
        stream = Stream()
        ring, mem = _ring_pair(batch=batch, stream=stream, prioritized_replay=True, beta_steps=4)
        net = _net(mode, batch=batch, stream=stream)
        random.seed(21)
        mem.seed_device_rng(random)
        if fused:
            net.train_fused(mem, 2)
            net.train_fused(mem, 3)
        else:
            for _ in range(5):
                mem.sample()
                net.train(DeviceMinibatch(mem, sampled=True))
        out.append((net.last_costs(5), _dev(mem, _L().PTR_INDEXES, np.int32, batch), mem.last_weights,
                    mem.priorities, _state(net)[0], device_tree(mem)[1]))
    for x, y in zip(out[0][:4], out[1][:4]):
        assert (x == y).all()
    for x, y in zip(out[0][4], out[1][4]):
        assert (x == y).all()
    for x, y in zip(out[0][5], out[1][5]):
        assert (x == y).all()
    assert (out[0][2] != F32(1)).any()


# ---------------------------------------------------------------------------------------------------- loop
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_agent_loop(mode):
    """The agent's loop (add frames, getMinibatch, train) with prioritized replay and the process-global `random`:
    every draw equals the oracle's draw on the device's tree, `random` matches the oracle's stream after every draw,
    and step_host on a twin ring and net gives the same costs, priorities and weights bit for bit."""
    from simple_dqn_b200 import Stream
    runs = []
    a, r, s, t = _frames(2000, 8, terminal_p=0.02)
    for use_step_host in (False, True):
        stream = Stream()
        mem = _mem(1500, batch=32, rng="python", stream=stream, prioritized_replay=True, beta_steps=5)
        net = _net(mode, stream=stream)
        mem.add_batch(a[:600], r[:600], s[:600], t[:600])
        random.seed(99)
        costs = []
        pos = 600
        for it in range(6):
            n = 4 + it                                       # env steps between train steps
            fa, fr, fs, ft = a[pos:pos + n], r[pos:pos + n], s[pos:pos + n], t[pos:pos + n]
            pos += n
            random.random()                                  # somebody else draws from `random` (exploration)
            if use_step_host:
                costs.extend(net.step_host(mem, fa, fr, fs, ft, train_repeat=1))
            else:
                for i in range(n):
                    mem.add(fa[i], fr[i], fs[i], ft[i])
                _, sums, mins, count = check_tree(mem)
                rng = MT19937.from_python(random)
                idx, w = P.draw(sums, mins, rng, 32, count, it, 0.4, 5)
                mb = mem.getMinibatch()
                pre = mb[0]                                  # looking at it draws on the spot (statistics.py:85)
                assert pre.shape == (32, 4, 84, 84)
                assert (mem.last_indexes == idx).all()
                assert list(random.getstate()[1]) == rng.state625()
                np.testing.assert_array_max_ulp(mem.last_weights, w, maxulp=2)
                net.train(mb)                                # a prioritized minibatch trains from the ring
                costs.append(net.last_costs(1)[0])
        runs.append((np.array(costs, F32), mem.priorities, mem.last_weights, _state(net)[0], random.getstate()))
    x, y = runs
    assert (x[0] == y[0]).all() and (x[1] == y[1]).all() and (x[2] == y[2]).all()
    for p, q in zip(x[3], y[3]):
        assert (p == q).all()
    assert x[4] == y[4]


# ---------------------------------------------------------------------------------------------------- off state
def test_off_state_and_refusals():
    from simple_dqn_b200 import DeviceMinibatch, Stream
    L = _L()
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    p, b = C.c_void_p(), C.c_size_t()
    for which in (L.PTR_PRIORITIES, L.PTR_SUM_TREE, L.PTR_IS_WEIGHTS, L.PTR_MAX_PRIORITY, L.PTR_MIN_TREE):
        L.call("b200dqn_replay_device_ptr", mem._h, which, C.byref(p), C.byref(b))
        assert p.value is None and b.value == 0          # nothing allocated while it was never on
    net = _net("tcgen05", stream=stream)
    random.seed(3)
    mem.seed_device_rng(random)
    net.train_fused(mem, 1)
    plain = net.launches_per_step()
    with pytest.raises(AssertionError):
        net.last_td_errors()                             # no prioritized step yet
    mem.set_prioritized(True)
    net.train_fused(mem, 1)                              # the graph is re-captured for the prioritized ring
    assert net.launches_per_step() == plain + 1          # the sampler is swapped, the priority update added
    mem.set_prioritized(False)
    net.train_fused(mem, 1)
    assert net.launches_per_step() == plain
    mb = mem.getMinibatch()
    assert not isinstance(mb, DeviceMinibatch)           # off: the host tuple, as before
    with pytest.raises(NotImplementedError, match="prioritized"):
        net.comm_init(bytes(128), 0, 2)              # this net has trained from a prioritized ring
