"""Random-shift augmentation on the device against tests/shift_oracle.py, on both engines and both schedules: the
device's offsets equal the stated draw exactly; every slot a train step runs (the online network on the prestates, the
target network on the poststates, Double DQN's online network on the poststates and the Munchausen pass on the
prestates) equals a twin without augmentation run on the host-shifted states, bit for bit, for the uniform, prioritized
and n-step rings, history lengths 1 to 16 and batch sizes on both sides of conv1's tile edges and of the conv23
threshold; a whole host-tuple step, with every head and target, equals the twin's step on the shifted tuple in every
weight, optimizer state, cost and readback, including at every corner offset of p = 8; predict never shifts; and five
fused steps follow the numpy step on the shifted minibatches."""
import random

import numpy as np
import pytest

import shift_oracle as SH
from helpers import make_args, rel_l2
from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring
from test_gpu_nstep import _mem

pytestmark = pytest.mark.gpu

F32 = np.float32
MODES = ["tcgen05", "fp32"]


def _stream(serial):
    from simple_dqn_b200 import Stream
    return None if serial else Stream()


def _net(mode, shift, A=4, batch=32, hist=4, stream=None, seed=3, **kw):
    """A net with scaled fc weights, small random optimizer states and target weights apart from the online ones; the
    same arguments with another `shift` make a twin with the same bits."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, history_length=hist, random_seed=seed, random_shift=shift, **kw),
                       math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [[np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for _ in range(net.num_states)]
                         for w in ws])
    tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws]
    if kw.get("target_steps", 10000):
        net.set_weights(tws, None, which=1)
    return net, ws, tws


def _minibatch(batch, hist, A, seed):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (batch, hist, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (batch, hist, 84, 84)).astype(np.uint8)
    return (pre, rs.randint(0, A, batch).astype(np.uint8), rs.randint(-3, 4, batch).astype(np.int64), post,
            rs.rand(batch) < 0.3)


def _eq(a, b, what):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and (a == b).all(), (what, int((a != b).sum()))


def _same_nets(a, b):
    for x, y in zip(a.get_weights(with_states=False), b.get_weights(with_states=False)):
        _eq(x, y, "weights")
    for x, y in zip(a.get_states(), b.get_states()):
        for p, q in zip(x, y):
            _eq(p, q, "states")


# readbacks of the stages each head keeps, compared between the augmented net and its twin after every step
READBACKS = {
    "scalar": ("last_deltas", "last_row_costs"),
    "double": ("last_online_postq", "last_deltas"),
    "c51": ("last_logits", "last_distributions", "last_target_distribution", "last_logit_grads"),
    "dueling": ("last_advantages", "last_values", "last_deltas"),
    "qr": ("last_quantiles", "last_target_quantiles", "last_quantile_grads"),
    "mdqn": ("last_target_q_pre", "last_td_targets", "last_deltas"),
    "iqn": ("last_taus", "last_iqn_quantiles", "last_iqn_target_quantiles", "last_iqn_quantile_grads"),
}
HEAD_ARGS = {
    "scalar": {},
    "double": {"double_dqn": True},
    "c51": {"distributional": True, "num_atoms": 51},
    "dueling": {"dueling": True},
    "qr": {"quantile_regression": True, "num_quantiles": 16},
    "mdqn": {"munchausen": True},
    "iqn": {"implicit_quantiles": True, "num_tau_samples": 8, "num_quantile_samples": 8},
}


def _pin_step(a, b, mb, pad, head="scalar"):
    """One host-tuple step of augmented net a and of twin b on the host-shifted tuple: the offsets are the stated draw
    and every cost, Q row, slot-0 activation, head readback, weight and optimizer state matches bit for bit."""
    c0 = a.shift_draws()
    a.train(mb)
    assert a.shift_draws() == c0 + 1
    off = a.last_shifts()
    _eq(off, SH.draw(a.shift_seed, c0, pad, a.batch_size), "offsets")
    b.train(SH.shift_minibatch(mb, off))
    _eq(a.last_costs(1), b.last_costs(1), "cost")
    for x, y in zip(a.last_q(), b.last_q()):
        _eq(x, y, "q")
    if head != "iqn":
        for x, y in zip(a.last_activations(), b.last_activations()):
            _eq(x, y, "h1..h4")
    for name in READBACKS[head]:
        _eq(getattr(a, name)(), getattr(b, name)(), name)
    _same_nets(a, b)
    return off


# ---------------------------------------------------------------------------------------------------- the draw
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("pad", [1, 4, 8])
def test_draw_equals_rule(mode, pad):
    """The device's (2, batch, 2) offsets equal rule 1 exactly at every batch size; the counter starts at 0 and every
    train step advances it by one (host tuple, train_fused(n) with step k drawing at counter k); predict touches
    nothing."""
    for batch in (1, 32, 33, 65, 257, 4096):
        stream = _stream(False)
        net, _, _ = _net(mode, pad, batch=batch, stream=stream)
        assert net.random_shift == pad and net.shift_draws() == 0
        z = np.zeros((batch, 4, 84, 84), np.uint8)
        mb = (z, np.zeros(batch, np.uint8), np.zeros(batch, np.int64), z, np.zeros(batch, np.bool_))
        net.train(mb)
        assert net.shift_draws() == 1
        _eq(net.last_shifts(), SH.draw(net.shift_seed, 0, pad, batch), ("offsets", batch))
        net.predict(z)
        assert net.shift_draws() == 1
        _eq(net.last_shifts(), SH.draw(net.shift_seed, 0, pad, batch), ("predict kept the offsets", batch))
        if batch <= 257:
            _, mem = _ring_pair(batch, 4, stream)
            random.seed(5)
            mem.seed_device_rng(random)
            net.train_fused(mem, 3)
            assert net.shift_draws() == 4
            _eq(net.last_shifts(), SH.draw(net.shift_seed, 3, pad, batch), ("fused step 3", batch))
            net.train_fused(mem, 1)
            _eq(net.last_shifts(), SH.draw(net.shift_seed, 4, pad, batch), ("fused step 4", batch))


def _ring_pair(batch, hist, stream, size=3000, seed=4, **kw):
    ring = ReplayOracle(size, history_length=hist, batch_size=batch)
    synthetic_ring(ring, seed=seed, block=100, terminal_p=0.05)
    mem = _mem(size, hist=hist, batch=batch, stream=stream, **kw)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    return ring, mem


# ---------------------------------------------------------------------------------------------------- slot pins
RINGS = [("uniform", {}), ("prioritized", {"prioritized_replay": True}), ("nstep", {"n_step": 3})]
HISTS = [1, 4, 5, 16]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("batch", [1, 32, 33, 64, 65, 256, 257])
def test_slot_pins_on_rings(mode, batch):
    """A Double DQN step trained from the ring (train_sampled): slot 0's Q row and H1..H4 equal the twin's predict on
    the prestates shifted by slot 0's offsets, slot 1's Q row the target twin's predict on the poststates shifted by
    slot 1's, and slot 2's Q row the twin's predict on those same shifted poststates.  The ring kind, history length
    and schedule rotate with the batch size."""
    from simple_dqn_b200 import DeviceMinibatch
    i = [1, 32, 33, 64, 65, 256, 257].index(batch) + (7 if mode == "fp32" else 0)
    kind, ring_kw = RINGS[i % 3]
    hist = HISTS[i % 4]
    stream = _stream(i % 2 == 1)
    pad = (4, 8, 1)[i % 3]
    a, ws, tws = _net(mode, pad, batch=batch, hist=hist, stream=stream, double_dqn=True)
    online, _, _ = _net(mode, 0, batch=batch, hist=hist, stream=stream)
    target, _, _ = _net(mode, 0, batch=batch, hist=hist, stream=stream)
    target.set_weights(tws, None)
    _, mem = _ring_pair(batch, hist, stream, **ring_kw)
    random.seed(9 + batch)
    mem.seed_device_rng(random)
    for step in range(2):
        mem.sample()
        pre, _, _, post, _ = (np.array(x) for x in mem._gather_to_host())
        c0 = a.shift_draws()
        ws_before = a.get_weights(with_states=False)
        a.train(DeviceMinibatch(mem, sampled=True))
        off = a.last_shifts()
        _eq(off, SH.draw(a.shift_seed, c0, pad, batch), ("offsets", kind, step))
        q0, q1 = a.last_q()
        h = a.last_activations()
        online.set_weights(ws_before, None)
        _eq(online.predict(SH.shift(pre, off[0])), q0, ("slot 0", kind, hist, step))
        for x, y in zip(online.last_activations(), h):
            _eq(x, y, ("slot 0 activations", kind, hist, step))
        _eq(target.predict(SH.shift(post, off[1])), q1, ("slot 1", kind, hist, step))
        _eq(online.predict(SH.shift(post, off[1])), a.last_online_postq(), ("slot 2", kind, hist, step))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("serial", [False, True])
def test_munchausen_pass_pin(mode, serial):
    """The Munchausen pass on the prestates reads slot 0's offsets: its Q row equals the target twin's predict on the
    prestates shifted by them."""
    stream = _stream(serial)
    for batch in (32, 65, 257):
        a, ws, tws = _net(mode, 4, batch=batch, stream=stream, munchausen=True)
        target, _, _ = _net(mode, 0, batch=batch, stream=stream)
        target.set_weights(tws, None)
        mb = _minibatch(batch, 4, 4, batch)
        a.train(mb)
        off = a.last_shifts()
        _eq(target.predict(SH.shift(mb[0], off[0])), a.last_target_q_pre(), ("pass", batch))


# ---------------------------------------------------------------------------------------------------- whole steps
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("head", list(HEAD_ARGS))
@pytest.mark.parametrize("serial", [False, True])
def test_whole_step_pin(mode, head, serial):
    """Three host-tuple steps, a target sync, and two more: the augmented net equals its twin trained on the shifted
    tuples in everything (for IQN the twin draws the same tau: same tau_seed, same counter history)."""
    stream = _stream(serial)
    batch = 33 if serial else 32
    a, _, _ = _net(mode, 4, batch=batch, stream=stream, **HEAD_ARGS[head])
    b, _, _ = _net(mode, 0, batch=batch, stream=stream, **HEAD_ARGS[head])
    for step in range(5):
        if step == 3:
            a.update_target_network()
            b.update_target_network()
        _pin_step(a, b, _minibatch(batch, 4, 4, 100 + step), 4, head)
    for x, y in zip(a.get_weights(which=1, with_states=False), b.get_weights(which=1, with_states=False)):
        _eq(x, y, "target weights")


@pytest.mark.parametrize("mode", MODES)
def test_edges_every_corner(mode):
    """p = 8 on frames whose every pixel differs from its neighbours: steps run until both slots have drawn all four
    corner offsets (+-8, +-8), and every step is pinned bit for bit to the twin on the shifted tuple."""
    batch = 257
    a, _, _ = _net(mode, 8, batch=batch, stream=_stream(False), double_dqn=True)
    b, _, _ = _net(mode, 0, batch=batch, stream=_stream(False), double_dqn=True)
    y, x = np.mgrid[0:84, 0:84]
    frame = ((y * 84 + x) * 37) % 251
    assert (np.diff(frame, axis=0) != 0).all() and (np.diff(frame, axis=1) != 0).all()
    rs = np.random.RandomState(0)
    seen = [set(), set()]
    corners = {(dy, dx) for dy in (-8, 8) for dx in (-8, 8)}
    for step in range(40):
        k = rs.randint(0, 251, (2, batch, 4, 1, 1))
        pre = ((frame[None, None] + k[0]) % 251).astype(np.uint8)
        post = ((frame[None, None] + k[1]) % 251).astype(np.uint8)
        mb = (pre, rs.randint(0, 4, batch).astype(np.uint8), rs.randint(-1, 2, batch).astype(np.int64), post,
              rs.rand(batch) < 0.2)
        off = _pin_step(a, b, mb, 8, "double")
        for z in range(2):
            seen[z] |= {tuple(o) for o in off[z]} & corners
        if seen[0] == corners and seen[1] == corners:
            break
    assert seen[0] == corners and seen[1] == corners, seen


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("serial", [False, True])
def test_ring_and_host_paths_agree(mode, serial):
    """With augmentation on, train_fused, sample() + train_sampled and the host tuple of the same minibatch give the
    same bits over three steps (the counter history is the same on all three nets)."""
    from simple_dqn_b200 import DeviceMinibatch
    stream = _stream(serial)
    nets = [_net(mode, 4, stream=stream)[0] for _ in range(3)]
    _, mem0 = _ring_pair(32, 4, stream)
    _, mem1 = _ring_pair(32, 4, stream)
    random.seed(3)
    mem0.seed_device_rng(random)
    random.seed(3)
    mem1.seed_device_rng(random)
    for _ in range(3):
        nets[0].train_fused(mem0, 1)
        mem1.sample()
        mb = tuple(np.array(x) for x in mem1._gather_to_host())
        nets[1].train(DeviceMinibatch(mem1, sampled=True))
        nets[2].train(mb)
    for other in nets[1:]:
        _eq(nets[0].last_costs(3), other.last_costs(3), "costs")
        _eq(nets[0].last_shifts(), other.last_shifts(), "offsets")
        _same_nets(nets[0], other)


# ---------------------------------------------------------------------------------------------------- predict
@pytest.mark.parametrize("mode", MODES)
def test_predict_never_shifts(mode):
    """predict on an augmented net is bit-identical to the plain twin's and touches no counter; the device pointers are
    EINVAL on a plain net; a fused step launches one kernel more; comm_init refuses."""
    from simple_dqn_b200 import _lib as L
    stream = _stream(False)
    a, _, _ = _net(mode, 4, stream=stream)
    b, _, _ = _net(mode, 0, stream=stream)
    s = _minibatch(32, 4, 4, 1)[0]
    _eq(a.predict(s), b.predict(s), "predict")
    assert a.shift_draws() == 0
    for which in (L.NET_PTR_SHIFT_OFFSETS, L.NET_PTR_SHIFT_DRAWS):
        with pytest.raises(AssertionError, match="random_shift"):
            b.device_view(which, (1,))
    _, mem = _ring_pair(32, 4, stream)
    random.seed(1)
    mem.seed_device_rng(random)
    for net in (a, b):
        net.train_fused(mem, 1)
    assert a.launches_per_step() == b.launches_per_step() + 1
    _eq(a.predict(s), a.predict(s), "predict twice")
    assert a.shift_draws() == 1
    with pytest.raises(NotImplementedError, match="random-shift"):
        a.comm_init(bytes(128), 0, 2)


# ---------------------------------------------------------------------------------------------------- trajectory
@pytest.mark.parametrize("mode", MODES)
def test_five_fused_steps_against_numpy(mode):
    """Five fused steps on a ring with p = 4 against the numpy step (oracle/dqn_oracle.py) on the host-shifted
    minibatches: the cost within 1e-3 and every layer within 2e-2 relative L2 of its change, the bars of the other
    feature tests."""
    size = 2000
    ring = ReplayOracle(size, batch_size=32)
    synthetic_ring(ring, seed=1, block=100, terminal_p=0.01)
    mem = _mem(size)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    net, ws, _ = _net(mode, 4)
    net.update_target_network()
    ws, ss = net.get_weights()
    orc = O.DQNOracle(4, weights=ws, states=ss)
    random.seed(11)
    rng = MT19937.from_python(random)
    mem.seed_device_rng(random)
    for _ in range(5):
        net.train_fused(mem, 1)
        off = net.last_shifts()
        ref = orc.train(SH.shift_minibatch(ring.getMinibatch(rng), off))
        cost = float(net.last_costs(1)[0])
        assert abs(cost - ref) <= 1e-3 * abs(ref), (cost, ref)
    w1 = net.get_weights(with_states=False)
    for layer in range(5):
        assert rel_l2(w1[layer] - ws[layer], orc.weights[layer] - ws[layer]) <= 2e-2 or \
            np.linalg.norm(w1[layer] - orc.weights[layer]) <= 2e-2 * np.linalg.norm(orc.weights[layer] - ws[layer]), \
            layer
