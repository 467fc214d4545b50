"""Double DQN target on the device (b200dqn_net_set_double_q) against the Double DQN oracle (tests/double_oracle.py).

Bars as in test_gpu_net.py: Q rows <= 1e-3 * max, cost rel 1e-3, gradients rel-L2 <= 2e-3, update rel-L2 <= 2e-2.
The device and the oracle compute Q to about 1e-3, so where two online Q values on a poststate are closer than that
they may pick different actions; the oracle then takes the device's choice (and the test checks that the two values
really are inside that band).  Bit-exact checks restate the head from the device's own Q rows.

An error in the third network slot alone (the online network on the poststates) would hide inside that 1e-3 band: its
only output is Q_online_post, which reaches the loss through an argmax.  So the slot is pinned bit for bit instead.
Every slot of a forward launch runs the same per-CTA code with no atomics, and the head sums the split-K partials in
slot-independent order, so slot 2 of a Double DQN step must equal slot 1 of a vanilla twin whose target network IS
the online network, at every batch-size dispatch, history length, engine and fc1 split count.  Where the Double DQN
target cannot differ from the vanilla one (all-terminal minibatches, one action), the whole step must be the vanilla
step bit for bit, which pins that the third slot clobbers no buffer the backward pass or the optimizer reads.
(The float64 bound on every kernel of a Double DQN step is in tests/test_gpu_kernels.py.)
"""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from double_oracle import DoubleDQNOracle, head_restated
from helpers import make_args, rel_l2
from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring
from test_gpu_kernels import SCHEDS, SWEEP

pytestmark = pytest.mark.gpu

F32 = np.float32


def _mb(n, num_actions, seed, hist=4, terminal_p=0.3, reward_range=(-3, 4)):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8)
    return (pre, rs.randint(0, num_actions, n).astype(np.uint8),
            rs.randint(reward_range[0], reward_range[1], n).astype(np.int64), post, rs.rand(n) < terminal_p)


def _stream(sched):
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


def _paired(num_actions, mode, batch=32, hist=4, stream=None, optimizer="rmsprop", seed=3, double=True, **kw):
    """Device net and Double DQN oracle with identical online weights and DIFFERENT target weights (the target is
    the online net one perturbation ago), so online and target prefer different poststate actions."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(num_actions, make_args(batch_size=batch, history_length=hist, random_seed=seed,
                                              optimizer=optimizer, double_dqn=double, **kw),
                       math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws]
    ss = [np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for w in ws]
    f = lambda scale, w, absolute=False: ((np.abs(rs.randn(*w.shape)) if absolute else rs.randn(*w.shape)) *
                                          scale).astype(F32)
    if optimizer == "adam":
        ss = [[f(1e-3, w), f(1e-5, w, True)] for w in ws]
    elif optimizer == "adadelta":
        ss = [[f(1e-5, w, True), f(1e-9, w, True), f(1e-4, w)] for w in ws]
    net.set_weights(ws, ss)
    if kw.get("target_steps", 10000):
        net.set_weights(tws, None, which=1)
    net.keep_grads(True)
    okw = {k: v for k, v in kw.items() if k in ("clip_error", "min_reward", "max_reward", "target_steps")}
    orc = DoubleDQNOracle(num_actions, double_dqn=double, batch_size=batch, weights=ws, states=ss,
                          optimizer=optimizer, **okw)
    if kw.get("target_steps", 10000):
        for t, w in zip(orc.target_weights, tws):
            t[...] = w
    return net, orc


def _first_max(q):
    return np.argmax(q, axis=1)


def _follow_device(dev_online_postq):
    """Oracle pick: its own first maximum, or the device's where the two differ by less than the 1e-3 band."""
    dev = _first_max(dev_online_postq)

    def pick(oq):
        a = _first_max(oq)
        rows = np.nonzero(a != dev)[0]
        band = 1e-3 * np.abs(oq).max()
        for i in rows:
            assert oq[i, a[i]] - oq[i, dev[i]] <= band, (i, oq[i], dev_online_postq[i])
        out = a.copy()
        out[rows] = dev[rows]
        return out
    return pick


CASES = [(4, 4), (18, 4), (32, 4), (4, 1), (4, 5)]   # (num_actions, history_length)


@pytest.mark.parametrize("mode,sched,batch", [("tcgen05", s, b) for s in ("serial", "branches") for b in (1, 32, 40, 256)] +
                         [("fp32", s, 32) for s in ("serial", "branches")])
@pytest.mark.parametrize("num_actions,hist", CASES)
def test_double_train_step_parity(mode, sched, batch, num_actions, hist):
    net, orc = _paired(num_actions, mode, batch=batch, hist=hist, stream=_stream(sched))
    mb = _mb(batch, num_actions, 2, hist=hist)
    w0 = [w.copy() for w in orc.weights]
    net.train(mb, 0)
    oq = net.last_online_postq()
    orc.pick = _follow_device(oq)
    ref_cost = orc.train(mb)
    L = orc.last
    preq, postq = net.last_q()
    assert np.abs(preq - L["preq"]).max() <= 1e-3 * np.abs(L["preq"]).max()
    assert np.abs(postq - L["postq"]).max() <= 1e-3 * np.abs(L["postq"]).max()
    assert np.abs(oq - L["online_postq"]).max() <= 1e-3 * np.abs(L["online_postq"]).max()
    cost = net.last_costs(1)[0]
    assert abs(cost - ref_cost) <= 1e-3 * abs(ref_cost)
    bars = [2e-3] * 5
    if mode == "fp32":
        # The SIMT engine's plain fp32 sums flip a few near-zero Rectlin masks against numpy's; on these weights its
        # vanilla step already sits at 1.7-1.9e-3 in the conv layers at H = 1.  The Double DQN step may take twice
        # what the vanilla step takes on the same weights and minibatch.
        van, vorc = _paired(num_actions, mode, batch=batch, hist=hist, stream=_stream(sched), double=False)
        van.train(mb, 0)
        vorc.train(mb)
        bars = [max(2e-3, 2 * rel_l2(g, r)) for g, r in zip(van.get_grads(), vorc.last["grads"])]
    for l, (g, r) in enumerate(zip(net.get_grads(), L["grads"])):
        assert rel_l2(g, r) <= bars[l], (l, rel_l2(g, r), bars[l])
    ws = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l
    if batch >= 32:   # the two networks disagree on some poststates: the Double DQN target is really in play
        assert (_first_max(postq) != _first_max(oq)).any()


@pytest.mark.parametrize("optimizer", ["adam", "adadelta"])
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_double_train_step_parity_other_optimizers(mode, optimizer):
    net, orc = _paired(6, mode, stream=_stream("branches"), optimizer=optimizer)
    mb = _mb(32, 6, 4)
    w0 = [w.copy() for w in orc.weights]
    net.train(mb, 0)
    orc.pick = _follow_device(net.last_online_postq())
    ref_cost = orc.train(mb)
    assert abs(net.last_costs(1)[0] - ref_cost) <= 1e-3 * abs(ref_cost)
    ws = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l


def _check_head_bits(net, mb, discount=0.99, min_reward=-1, max_reward=1, clip=1.0):
    """deltas, dZ4 and the batch cost restated from the device's own preq, postq and Q_online_post."""
    preq, postq = net.last_q()
    oq = net.last_online_postq()
    pre, act, rew, post, term = mb
    deltas, row_cost = head_restated(preq, postq, oq, act, rew, term, discount, min_reward, max_reward, clip)
    assert (net.last_deltas() == deltas).all()
    h4 = net.last_activations()[3]
    d = deltas[np.arange(len(act)), act]
    dz4 = np.where(h4 > 0, d[:, None] * net._w5_before[act], F32(0)).astype(F32)
    assert (net.last_dz()[3] == dz4).all()
    tot = F32(0)
    for c in row_cost:
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(len(act)))


@pytest.mark.parametrize("case", ["all_terminal", "no_terminal", "asymmetric_clip", "no_error_clip"])
def test_double_head_bit_exact(case):
    kw = dict(all_terminal=dict(), no_terminal=dict(), asymmetric_clip=dict(min_reward=-2, max_reward=1),
              no_error_clip=dict(clip_error=0))[case]
    net, _ = _paired(18, "tcgen05", stream=_stream("branches"), **kw)
    p = dict(all_terminal=1.0, no_terminal=0.0).get(case, 0.3)
    mb = _mb(32, 18, 6, terminal_p=p, reward_range=(-4, 5))
    net._w5_before = net.get_weights(with_states=False)[4].copy()   # the W5 the head reads (train updates it)
    net.train(mb, 0)
    _check_head_bits(net, mb, min_reward=kw.get("min_reward", -1), max_reward=kw.get("max_reward", 1),
                     clip=float(kw.get("clip_error", 1.0)))


def test_double_exact_tie_takes_first_index():
    """Online W5 rows 0 and 1 are identical and dominate, so Q_online(s', 0) == Q_online(s', 1) exactly and
    a* must be 0; the target rows differ, so taking action 1 would change the deltas."""
    net, _ = _paired(4, "tcgen05", stream=_stream("branches"))
    ws, ss = net.get_weights()
    tws = net.get_weights(which=1, with_states=False)
    ws[4][0] = ws[4][1] = np.abs(ws[4][0]) * F32(4)
    tws[4][0], tws[4][1] = np.abs(tws[4][0]) * F32(2), -np.abs(tws[4][1])
    net.set_weights(ws, ss)
    net.set_weights(tws, None, which=1)
    mb = _mb(32, 4, 8, terminal_p=0.0)
    net._w5_before = ws[4].copy()
    net.train(mb, 0)
    preq, postq = net.last_q()
    oq = net.last_online_postq()
    assert (oq[:, 0] == oq[:, 1]).all() and (_first_max(oq) == 0).all()
    assert (postq[:, 0] != postq[:, 1]).all()
    _check_head_bits(net, mb)
    wrong = oq.copy()
    wrong[:, 1] = np.nextafter(wrong[:, 1], F32(np.inf))
    d_wrong, _ = head_restated(preq, postq, wrong, mb[1], mb[2], mb[4])
    assert (d_wrong != net.last_deltas()).any()


def _state(net):
    ws, _ = net.get_weights()
    return ws, net.get_states(), net.get_weights(which=1, with_states=False)


def _assert_same(a, b):
    for x, y in zip(a, b):
        if isinstance(x, (list, tuple)):
            _assert_same(x, y)
        else:
            assert (x == y).all()


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_double_equals_vanilla_with_equal_weights_and_after_switching_off(mode):
    """Equal online and target weights: a* is the argmax of the same row, so the first (Double DQN) fused step is the
    vanilla step bit for bit.  Then double Q goes off: the captured graph must be rebuilt, and the next steps (online
    and target now differ) are vanilla steps again."""
    from simple_dqn_b200 import ReplayMemory, Stream
    ring = ReplayOracle(3000, batch_size=32)
    synthetic_ring(ring, seed=9, block=150, terminal_p=0.02)
    runs = []
    for double in (False, True):
        stream = Stream()
        mem = ReplayMemory(3000, make_args(), rng="device", stream=stream)
        mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
        mem.set_cursor(ring.count, ring.current)
        net, _ = _paired(6, mode, stream=stream, double=double)
        net.update_target_network()
        random.seed(21)
        mem.seed_device_rng(random)
        net.train_fused(mem, 1)
        first = (net.last_costs(1), net.last_deltas(), _state(net))
        if double:
            net.set_double_dqn(False)
        net.train_fused(mem, 2)
        runs.append((first, net.last_costs(3), _state(net)))
    (fa, ca, sa), (fb, cb, sb) = runs
    assert (fa[0] == fb[0]).all() and (fa[1] == fb[1]).all()
    _assert_same(fa[2], fb[2])
    assert (ca == cb).all()
    _assert_same(sa, sb)


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_double_equals_vanilla_at_target_steps_zero(mode):
    outs = []
    for double in (False, True):
        net, _ = _paired(4, mode, stream=_stream("branches"), double=double, target_steps=0)
        for i in range(3):
            net.train(_mb(32, 4, 30 + i), 0)
        outs.append((net.last_costs(3), net.last_deltas(), _state(net), net))
    (ca, da, sa, _), (cb, db, sb, nb) = outs
    assert (ca == cb).all() and (da == db).all()
    _assert_same(sa, sb)
    assert (nb.last_online_postq() == nb.last_q()[1]).all()   # one network: Q_online_post is the postq row


FUSED_CASES = ([("tcgen05", 32, 4), ("fp32", 32, 4), ("tcgen05", 65, 4), ("tcgen05", 257, 4)] +
               [("tcgen05", 32, h) for h in (1, 5, 16)] + [("fp32", 65, 4)])


@pytest.mark.parametrize("mode,batch,hist", FUSED_CASES,
                         ids=[m if (b, h) == (32, 4) else "%s-b%d-h%d" % (m, b, h) for m, b, h in FUSED_CASES])
def test_double_fused_ring_equals_host_minibatch(mode, batch, hist):
    """Batches 65 and 257 cross the two-kernel conv forward and the 4-split fc1 with three slots; H = 16 refills
    conv1's frame ring across three slots of CTAs."""
    from simple_dqn_b200 import ReplayMemory, Stream
    ring = ReplayOracle(4000, history_length=hist, batch_size=batch)
    synthetic_ring(ring, seed=4, block=200, terminal_p=0.02)
    nets = []
    for fused in (True, False):
        stream = Stream() if fused else None
        mem = ReplayMemory(4000, make_args(batch_size=batch, history_length=hist), rng="device", stream=stream)
        mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
        mem.set_cursor(ring.count, ring.current)
        net, _ = _paired(4, mode, batch=batch, hist=hist, stream=stream)
        random.seed(77)
        mem.seed_device_rng(random)
        if fused:
            net.train_fused(mem, nsteps=2)
            net.train_fused(mem, nsteps=3)
        else:
            for _ in range(5):
                net.train(mem.getMinibatch(), 0)
        nets.append(net)
    nf, nu = nets
    assert np.allclose(nf.last_costs(5), nu.last_costs(5), rtol=1e-6)
    _assert_same(_state(nf), _state(nu))


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_double_device_minibatch_step_host_and_trajectory(mode):
    """DeviceMinibatch (trained in place from the ring, lock-step python `random`), then step_host, then fused
    steps: a 5-step trajectory against the Double DQN oracle on the same minibatches, with a per-step cost trace."""
    from simple_dqn_b200 import DeviceMinibatch, ReplayMemory, Stream
    ring = ReplayOracle(3000, batch_size=32)
    synthetic_ring(ring, seed=6, block=100, terminal_p=0.02)
    stream = Stream()
    mem = ReplayMemory(3000, make_args(), rng="python", device_minibatch=True, stream=stream)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    net, orc = _paired(4, mode, stream=stream)
    w0 = [w.copy() for w in orc.weights]
    random.seed(5)
    rng = MT19937.from_python(random)
    costs, ref = [], []
    mb = mem.getMinibatch()
    assert isinstance(mb, DeviceMinibatch)
    net.train(mb, 0)
    costs.append(net.last_costs(1)[0])
    orc.pick = _follow_device(net.last_online_postq())
    ref.append(orc.train(ring.getMinibatch(rng)))
    empty = np.zeros((0,) + tuple(mem.dims), np.uint8)
    for _ in range(4):
        costs.extend(net.step_host(mem, [], [], empty, [], train_repeat=1))
        orc.pick = _follow_device(net.last_online_postq())
        ref.append(orc.train(ring.getMinibatch(rng)))
    rel = np.abs(np.array(costs) - np.array(ref)) / np.abs(ref)
    assert rel.max() <= 2e-3, rel
    ws = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l


def test_double_comm_init_refused():
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(4, make_args(double_dqn=True), math_mode="tcgen05")
    with pytest.raises(NotImplementedError, match="Double DQN"):
        net.comm_init(bytes(128), 0, 2)
    net.set_double_dqn(False)
    assert not net.double_dqn


def _twins(num_actions, mode, batch, hist, sched, **kw):
    """N (Double DQN, online W, target T != W), V1 (vanilla, W and T) and V2 (vanilla, W and W): all weights set
    from the host, so every tile image comes from the pack kernels."""
    n, _ = _paired(num_actions, mode, batch=batch, hist=hist, stream=_stream(sched), **kw)
    v1, _ = _paired(num_actions, mode, batch=batch, hist=hist, stream=_stream(sched), double=False, **kw)
    v2, _ = _paired(num_actions, mode, batch=batch, hist=hist, stream=_stream(sched), double=False, **kw)
    v2.set_weights(v2.get_weights(with_states=False), None, which=1)
    return n, v1, v2


def _assert_slot_identity(mode, batch, hist=4, num_actions=4, sched="branches"):
    """Slots 0 and 1 of N are V1's; slot 2 of N (Q_online_post) is V2's slot 1, on the same poststates.  Three steps:
    before steps 2 and 3 V2 is reloaded with N's updated fp32 weights (both of its networks), so N's
    optimizer-refreshed online tile images must equal a fresh pack of the same weights, in slot 0 and in slot 2."""
    n, v1, v2 = _twins(num_actions, mode, batch, hist, sched)
    for step in range(3):
        mb = _mb(batch, num_actions, 40 + step, hist=hist)
        assert (mb[0] != mb[3]).any()
        if step > 0:
            ws = n.get_weights(with_states=False)
            v2.set_weights(ws, None)
            v2.set_weights(ws, None, which=1)
        n._w5_before = n.get_weights(with_states=False)[4].copy()
        for net in (n, v1, v2) if step == 0 else (n, v2):
            net.train(mb, 0)
        preq, postq = n.last_q()
        oq = n.last_online_postq()
        vpre, vpost = v2.last_q()
        assert (oq == vpost).all(), (step, np.abs(oq - vpost).max())
        assert (preq == vpre).all(), (step, np.abs(preq - vpre).max())
        _check_head_bits(n, mb)
        if step == 0:
            v1pre, v1post = v1.last_q()
            assert (preq == v1pre).all() and (postq == v1post).all()
            for h, hv in zip(n.last_activations(), v1.last_activations()):
                assert (h == hv).all()
            if batch >= 32 and num_actions > 1:     # online and target disagree: the slot decides some targets
                assert (_first_max(oq) != _first_max(postq))[~mb[4]].any()


SLOT_CASES = ([("tcgen05", s, b, 4, 4) for s in SCHEDS for b in SWEEP] +
              [("tcgen05", "branches", b, h, 4) for h in (1, 5, 16) for b in (1, 64, 65)] +
              [("tcgen05", "branches", 33, 4, a) for a in (1, 18)] +
              [("fp32", "serial", b, 4, 4) for b in (1, 32, 65)])


@pytest.mark.parametrize("mode,sched,batch,hist,num_actions", SLOT_CASES)
def test_double_third_slot_is_the_online_forward(mode, sched, batch, hist, num_actions):
    _assert_slot_identity(mode, batch, hist, num_actions, sched)


@pytest.mark.parametrize("splits", [1, 4, 14])
def test_double_third_slot_under_forced_fc1_splits(splits):
    """B200DQN_FC1_SPLITS is read once per process, so the check runs in a child process."""
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_double as T\n"
            "for batch in (33, 257):\n"
            "    T._assert_slot_identity('tcgen05', batch)\n"
            "print('SLOTS OK')\n" % (ROOT, os.path.join(ROOT, "tests")))
    env = dict(os.environ, B200DQN_FC1_SPLITS=str(splits))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    assert "SLOTS OK" in out.stdout


VANILLA_CASES = ([(m, s, b, "all_terminal") for m in ("tcgen05", "fp32") for s in SCHEDS for b in SWEEP] +
                 [("tcgen05", "branches", 33, "adam"), ("fp32", "branches", 33, "adam")] +
                 [("tcgen05", "branches", b, "one_action") for b in (1, 33, 65, 257)] +
                 [("fp32", "serial", b, "one_action") for b in (1, 33)])


@pytest.mark.parametrize("mode,sched,batch,case", VANILLA_CASES)
def test_double_step_is_vanilla_where_the_target_cannot_differ(mode, sched, batch, case):
    """All-terminal minibatches (the target ignores Q) and A = 1 (a* = 0 is the maximum), with T != W: two Double DQN
    steps equal two vanilla steps bit for bit (costs, deltas, gradients, online and target weights, every optimizer
    state plane), although the Double DQN step runs the third slot in every forward launch."""
    num_actions, terminal_p = (1, 0.0) if case == "one_action" else (4, 1.0)
    optimizer = "adam" if case == "adam" else "rmsprop"
    runs = []
    for double in (False, True):
        net, _ = _paired(num_actions, mode, batch=batch, stream=_stream(sched), optimizer=optimizer, double=double)
        steps = []
        for i in range(2):
            net.train(_mb(batch, num_actions, 50 + i, terminal_p=terminal_p), 0)
            steps.append((net.last_deltas(), net.get_grads()))
        runs.append((net.last_costs(2), steps, _state(net)))
        if double:      # the third slot really ran, with the online weights
            assert (net.last_online_postq() != net.last_q()[1]).any()
    (ca, sa, wa), (cb, sb, wb) = runs
    assert (ca == cb).all(), (ca, cb)
    _assert_same(sa, sb)
    _assert_same(wa, wb)


def _live_net(ring, mode, double_at_creation, make=None):
    """make(stream, double): the net (batch 32, H = 4); by default _paired's with six actions."""
    from simple_dqn_b200 import ReplayMemory, StateBuffer, Stream
    stream = Stream()
    mem = ReplayMemory(ring.size, make_args(), rng="device", stream=stream)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    net = make(stream, double_at_creation) if make else _paired(6, mode, stream=stream, double=double_at_creation)[0]
    if double_at_creation:
        net.set_double_dqn(False)       # the third slot's buffers exist; the steps below start vanilla
    random.seed(21)
    mem.seed_device_rng(random)
    return net, mem, StateBuffer(make_args(), stream=stream)


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_double_switched_on_live_equals_switched_on_at_creation(mode):
    """A is created vanilla, runs fused-step graphs and the state-window predict graph, then switches Double DQN on,
    which reallocates the fc1 partials those graphs hold; B allocated the third slot at creation.  Every cost, weight,
    optimizer state and fast-path Q row must agree, also across A switching off and on again, toggling keep_grads and
    a target sync in the middle of the run; the fast-path Q equals host predict on the same window."""
    assert_switched_on_live_equals_at_creation(mode)


def assert_switched_on_live_equals_at_creation(mode, make=None):
    """The run of test_double_switched_on_live_equals_switched_on_at_creation on the nets make(stream, double)
    builds (_live_net)."""
    ring = ReplayOracle(3000, batch_size=32)
    synthetic_ring(ring, seed=12, block=150, terminal_p=0.02)
    frames = np.random.RandomState(0).randint(0, 256, (8, 84, 84)).astype(np.uint8)
    nets = [_live_net(ring, mode, at_creation, make) for at_creation in (False, True)]
    n_frames = [0]

    def predict_both():
        qs = []
        for net, _, buf in nets:
            for i in range(n_frames[0], n_frames[0] + 2):
                buf.add(frames[i])
            states = buf.getStateMinibatch()
            q = net.predict(states)             # the captured predict graph
            host = net.predict(np.asarray(states))
            assert (q[0] == host[0]).all() and not q[1:].any()
            qs.append(q)
        n_frames[0] += 2
        assert (qs[0] == qs[1]).all()

    def train_both(k, total):
        for net, mem, _ in nets:
            net.train_fused(mem, k)
        (a, _, _), (b, _, _) = nets
        assert (a.last_costs(total) == b.last_costs(total)).all()
        _assert_same(_state(a), _state(b))

    (a, _, _), (b, _, _) = nets
    train_both(2, 2)
    predict_both()
    for net in (a, b):
        net.set_double_dqn(True)
    train_both(2, 4)
    predict_both()
    assert (a.last_online_postq() == b.last_online_postq()).all()
    a.set_double_dqn(False)
    a.set_double_dqn(True)
    train_both(1, 5)
    a.keep_grads(False)
    train_both(1, 6)
    a.keep_grads(True)
    for net in (a, b):
        net.update_target_network()
    train_both(2, 8)
    predict_both()
    assert (a.last_online_postq() == b.last_online_postq()).all()
    assert (a.last_online_postq() != a.last_q()[1]).any()      # still a Double DQN step: T != W after the sync
