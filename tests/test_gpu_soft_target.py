"""The soft (Polyak-averaged) target update on the device against tests/soft_target_oracle.py, bit for bit, on both
engines: every target layer after a step is the rule applied to the device's own pre-step target and post-step online
weights, under every head, Double DQN, Munchausen, a prioritized n-step ring and random shifts, and the target's
optimizer states do not move.  A twin net loaded with the blended weights takes the same next step (so the tensor-core
target images equal a fresh pack of the fp32 target).  Also tau = 1 against a hard copy after every step, the train
entry points, the manual entry, the launch count and the refusals."""
import random

import numpy as np
import pytest

import soft_target_oracle as SOFT
from helpers import make_args
from test_gpu_distributional import _L, _ring_pair

pytestmark = pytest.mark.gpu

F32 = np.float32
MODES = ["tcgen05", "fp32"]


def _snet(mode, tau, stream=None, batch=32, hist=4, seed=3, optimizer="rmsprop", **kw):
    """A net with distinct online and target weights and nonzero optimizer states in every layer."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(4, make_args(batch_size=batch, history_length=hist, random_seed=seed, optimizer=optimizer,
                                    soft_target_tau=tau, **kw), math_mode=mode, stream=stream)
    rs = np.random.RandomState(seed)
    ws = net.get_weights(with_states=False)
    ws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.01)).astype(F32) if not np.abs(w).max() else w for w in ws]
    ws[3] = ws[3] * F32(3)
    net.set_weights(ws, [[np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for _ in range(net.num_states)]
                         for w in ws])
    net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                    [[np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for _ in range(net.num_states)] for w in ws],
                    which=1)
    return net


def _bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def _check_rule(net, tw_before, ts_before, tau):
    """get_weights(1) of every layer is the rule on the pre-step target and the post-step online weights, bit for bit;
    the target's state planes are unchanged."""
    ws = net.get_weights(with_states=False)
    tws = net.get_weights(which=1, with_states=False)
    assert len(tws) == len(tw_before)
    for layer, (got, exp) in enumerate(zip(tws, SOFT.blend_layers(tw_before, ws, tau))):
        assert (_bits(got) == _bits(exp)).all(), layer
    for layer, (got, exp) in enumerate(zip(net.get_states(which=1), ts_before)):
        for k, (g, e) in enumerate(zip(got, exp)):
            assert (_bits(g) == _bits(e)).all(), (layer, k)


HEADS = {
    "scalar": {}, "double": {"double_dqn": True}, "dueling": {"dueling": True},
    "c51": {"distributional": True, "num_atoms": 51}, "qr": {"quantile_regression": True, "num_quantiles": 32},
    "iqn": {"implicit_quantiles": True, "num_tau_samples": 8, "num_quantile_samples": 8},
    "fqf": {"fqf": True, "num_fractions": 8}, "rem": {"rem": True, "num_heads": 4},
    "boot": {"bootstrapped": True, "bootstrap_heads": 4, "bootstrap_p": 0.5}, "munchausen": {"munchausen": True},
    "per_nstep": {}, "shift": {"random_shift": 4},
}


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
@pytest.mark.parametrize("head", sorted(HEADS))
def test_one_step_applies_the_rule_to_every_layer(mode, sched, head):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream() if sched == "branches" else None
    per = head == "per_nstep"
    _, mem = _ring_pair(stream=stream, prioritized_replay=per, beta0=0.4)
    if per:
        mem.set_n_step(3)
    tau = 0.005 if head != "scalar" else 0.3
    net = _snet(mode, tau, stream=stream, **HEADS[head])
    assert net.soft_target_tau == tau
    for step in range(2):
        tw, _ = net.get_weights(which=1)
        ts = net.get_states(which=1)
        idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
        mem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        _check_rule(net, tw, ts, tau)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("batch", [32, 128])
@pytest.mark.parametrize("hist", [1, 4])
def test_twin_loaded_with_the_blended_weights_takes_the_same_step(mode, batch, hist):
    """After k soft steps, a second net loaded with the first one's online and target weights and states takes the
    next step bit for bit like the first: costs, both Q rows (the target's row reads the target images on the
    tensor-core engine), online and target weights."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream, tstream = Stream(), Stream()
    _, mem = _ring_pair(batch=batch, hist=hist, stream=stream)
    _, tmem = _ring_pair(batch=batch, hist=hist, stream=tstream)
    net = _snet(mode, 0.05, stream=stream, batch=batch, hist=hist)
    for step in range(3):
        mem.set_indexes(np.array(random.Random(step).sample(range(50, 2900), batch), np.int32))
        net.train(DeviceMinibatch(mem, sampled=True))
    twin = _snet(mode, 0.05, stream=tstream, batch=batch, hist=hist, seed=11)
    for which in (0, 1):
        ws = net.get_weights(which=which, with_states=False)
        twin.set_weights(ws, net.get_states(which=which), which=which)
    idx = np.array(random.Random(9).sample(range(50, 2900), batch), np.int32)
    mem.set_indexes(idx)
    tmem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    twin.train(DeviceMinibatch(tmem, sampled=True))
    assert (_bits(net.last_costs(1)) == _bits(twin.last_costs(1))).all()
    for a, b in zip(net.last_q(), twin.last_q()):
        assert (_bits(a) == _bits(b)).all()
    for which in (0, 1):
        for a, b in zip(net.get_weights(which=which, with_states=False),
                        twin.get_weights(which=which, with_states=False)):
            assert (_bits(a) == _bits(b)).all()


@pytest.mark.parametrize("mode", MODES)
def test_tau_one_equals_a_hard_copy_after_every_step(mode):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream, tstream = Stream(), Stream()
    _, mem = _ring_pair(stream=stream)
    _, tmem = _ring_pair(stream=tstream)
    net = _snet(mode, 1.0, stream=stream)
    hard = _snet(mode, 0.0, stream=tstream)
    for step in range(4):
        idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
        mem.set_indexes(idx)
        tmem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        hard.train(DeviceMinibatch(tmem, sampled=True))
        hard.update_target_network()
        assert (_bits(net.last_costs(1)) == _bits(hard.last_costs(1))).all(), step
        for a, b in zip(net.get_weights(with_states=False), hard.get_weights(with_states=False)):
            assert (_bits(a) == _bits(b)).all(), step
        for a, b in zip(net.get_weights(which=1, with_states=False), hard.get_weights(which=1, with_states=False)):
            assert (a == b).all(), step


@pytest.mark.parametrize("mode", MODES)
def test_train_fused_n_equals_n_single_steps(mode):
    from simple_dqn_b200 import Stream
    stream, tstream = Stream(), Stream()
    _, mem = _ring_pair(stream=stream)
    _, tmem = _ring_pair(stream=tstream)
    net = _snet(mode, 0.01, stream=stream)
    twin = _snet(mode, 0.01, stream=tstream)
    random.seed(4)
    mem.seed_device_rng(random)
    key = mem.read_device_rng()
    _L().call("b200dqn_replay_set_rng", tmem._h, _L().np_ptr(key), tmem._stream)
    tmem._rng_on_device = True
    net.train_fused(mem, 5)
    for _ in range(5):
        twin.train_fused(tmem, 1)
    assert (_bits(net.last_costs(5)) == _bits(twin.last_costs(5))).all()
    for which in (0, 1):
        for a, b in zip(net.get_weights(which=which, with_states=False),
                        twin.get_weights(which=which, with_states=False)):
            assert (_bits(a) == _bits(b)).all()


@pytest.mark.parametrize("mode", MODES)
def test_step_host_and_host_tuple_train_blend(mode):
    from helpers import random_minibatch
    from simple_dqn_b200 import Stream
    stream = Stream()
    _, mem = _ring_pair(stream=stream)
    net = _snet(mode, 0.02, stream=stream)
    tw, _ = net.get_weights(which=1)
    ts = net.get_states(which=1)
    empty = np.zeros((0,) + tuple(mem.dims), np.uint8)
    net.step_host(mem, np.zeros(0, np.uint8), np.zeros(0, np.int64), empty, np.zeros(0, np.uint8), train_repeat=1)
    _check_rule(net, tw, ts, 0.02)
    tw, _ = net.get_weights(which=1)
    net.train(random_minibatch(32, 4, 5))
    _check_rule(net, tw, ts, 0.02)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("head", ["scalar", "fqf"])
def test_manual_entry_applies_the_rule_once(mode, head):
    """update_target_network(tau) on a net without a per-step blend: one application of the rule to every layer, the
    states untouched; update_target_network() is still the hard copy."""
    net = _snet(mode, 0.0, **({"fqf": True, "num_fractions": 8} if head == "fqf" else {}))
    tw, _ = net.get_weights(which=1)
    ts = net.get_states(which=1)
    net.update_target_network(0.25)
    _check_rule(net, tw, ts, 0.25)
    net.update_target_network()
    for a, b in zip(net.get_weights(with_states=False), net.get_weights(which=1, with_states=False)):
        assert (_bits(a) == _bits(b)).all()
    for bad in (0.0, -0.5, 1.5, float("nan")):
        with pytest.raises(AssertionError, match="tau"):
            net.update_target_network(bad)
    alias = _snet_alias(mode)
    with pytest.raises(AssertionError, match="target_steps = 0"):
        alias.update_target_network(0.5)


def _snet_alias(mode):
    from simple_dqn_b200 import DeepQNetwork
    return DeepQNetwork(4, make_args(target_steps=0), math_mode=mode)


@pytest.mark.parametrize("mode", MODES)
def test_manual_entry_rebuilds_the_target_images(mode):
    """After update_target_network(tau), a train step equals the step of a twin whose target was loaded from the host
    (a fresh pack of the blended fp32 weights)."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream, tstream = Stream(), Stream()
    _, mem = _ring_pair(stream=stream)
    _, tmem = _ring_pair(stream=tstream)
    net = _snet(mode, 0.0, stream=stream)
    net.update_target_network(0.4)
    twin = _snet(mode, 0.0, stream=tstream, seed=8)
    for which in (0, 1):
        twin.set_weights(net.get_weights(which=which, with_states=False), net.get_states(which=which), which=which)
    idx = np.array(random.Random(2).sample(range(50, 2900), 32), np.int32)
    mem.set_indexes(idx)
    tmem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    twin.train(DeviceMinibatch(tmem, sampled=True))
    for a, b in zip(net.last_q(), twin.last_q()):
        assert (_bits(a) == _bits(b)).all()
    assert (_bits(net.last_costs(1)) == _bits(twin.last_costs(1))).all()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("head", ["scalar", "c51", "iqn", "fqf"])
def test_launch_count_grows_by_the_documented_blends(mode, head):
    """One blend per update launch: conv1, conv2, conv3 and fc1 (with the SIMT engine's scalar fc2), fc2 on its own
    (tensor-core engine, or a per-action head), the embedding (IQN, FQF) and the fraction layer (FQF); in the static
    count before the first fused step and in the count taken while the step graph is captured."""
    from simple_dqn_b200 import Stream
    stream = Stream()
    _, mem = _ring_pair(stream=stream)
    random.seed(1)
    mem.seed_device_rng(random)
    tc = mode == "tcgen05"
    extra = 4 + (1 if tc or head != "scalar" else 0) + (1 if head in ("iqn", "fqf") else 0) + (head == "fqf")
    static, captured = [], []
    for tau in (0.0, 0.005):
        net = _snet(mode, tau, stream=stream, **HEADS[head])
        static.append(net.launches_per_step())
        net.train_fused(mem, 1)
        captured.append(net.launches_per_step())
    assert static[1] - static[0] == extra, static
    assert captured[1] - captured[0] == extra, captured


def test_comm_init_refuses():
    net = _snet("tcgen05", 0.005)
    with pytest.raises(NotImplementedError, match="soft target"):
        net.comm_init(bytes(128), 0, 2)
