"""GPU parity of the network half against the numpy oracle (oracle/dqn_oracle.py).

Tolerances (north_star: "Q-values within 1e-3 rel on identical fp32 weights/inputs"):
  * Q-values:        max|dQ| <= 1e-3 * max|Q|          (both math modes; fp32 mode is ~1e-5)
  * cost:            rel 1e-3
  * gradients:       rel-L2 <= 2e-3 per layer  (L2, not max: one ReLU-mask flip at a ~0
                     pre-activation is a legitimate fp32 reassociation effect, see
                     tests/test_oracle_dqn.py)
  * weights after k RMSProp steps: rel-L2 of the UPDATE (W_k - W_0) <= 2e-2
"""
import os
import pickle
import random

import numpy as np
import pytest

from helpers import make_args, random_minibatch, rel_l2
from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tcgen05"]


def _net(num_actions, mode, stream=None, **kw):
    from simple_dqn_b200 import DeepQNetwork
    try:
        return DeepQNetwork(num_actions, make_args(**kw), math_mode=mode, stream=stream)
    except NotImplementedError as e:
        pytest.skip(str(e))


def _stream(sched):
    """"serial": legacy default stream (plain serial launches, generic k_optimizer); "branches": a library
    stream, i.e. the PRODUCTION schedule — side-stream branches, PDL chain, fused per-layer optimizers."""
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


SCHEDS = ["serial", "branches"]


def _paired(num_actions, mode, seed=3, batch=32, stream=None, optimizer="rmsprop"):
    """A device net and an oracle net holding identical fp32 weights (trained-looking scale)."""
    net = _net(num_actions, mode, stream=stream, batch_size=batch, random_seed=seed, optimizer=optimizer)
    ws, ss = net.get_weights()
    # Xavier weights give Q ~ 1e-2; scale the last layers so Q ~ O(1) like a trained net
    ws[3] = ws[3] * np.float32(3.0)
    ws[4] = ws[4] * np.float32(3.0)
    rs = np.random.RandomState(seed)
    ss = [np.abs(rs.randn(*w.shape)).astype(np.float32) * np.float32(1e-4) for w in ws]
    f = lambda scale, w, absolute=False: ((np.abs(rs.randn(*w.shape)) if absolute else rs.randn(*w.shape)) *
                                          scale).astype(np.float32)
    if optimizer == "adam":         # Neon states [m, v]
        ss = [[f(1e-3, w), f(1e-5, w, True)] for w in ws]
    elif optimizer == "adadelta":   # Neon states [E[g^2], E[dx^2], dx]
        ss = [[f(1e-5, w, True), f(1e-9, w, True), f(1e-4, w)] for w in ws]
    net.set_weights(ws, ss)
    net.update_target_network()
    net.keep_grads(True)            # the fp32 dZ copies as well as the fp16 planes
    orc = O.DQNOracle(num_actions, batch_size=batch, weights=ws, states=ss, optimizer=optimizer)
    return net, orc


@pytest.mark.parametrize("mode", MODES)
def test_xavier_init_matches_oracle_draw_order(mode):
    net = _net(4, mode, random_seed=11)
    ws, ss = net.get_weights()
    ref = O.xavier_init(4, seed=11)
    assert all((a == b).all() for a, b in zip(ws, ref))
    assert all(not s.any() for s in ss)
    assert [w.shape for w in ws] == O.layer_shapes(4)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("num_actions,batch", [(4, 32), (18, 32), (4, 1), (6, 8), (4, 40), (4, 64), (4, 65), (4, 256),
                                               (4, 257)])
def test_predict_parity(mode, num_actions, batch):
    """net_create takes any batch 1..4096 (tile tails, partial M tiles): every size is held to the same bar."""
    net, orc = _paired(num_actions, mode, batch=batch)
    states = random_minibatch(batch, num_actions, 1)[0]
    q = net.predict(states)
    ref = orc.predict(states)
    assert q.shape == (batch, num_actions) and q.dtype == np.float32
    assert np.abs(q - ref).max() <= 1e-3 * np.abs(ref).max(), np.abs(q - ref).max() / np.abs(ref).max()
    if batch > 5:
        with pytest.raises(AssertionError):
            net.predict(states[:5])                             # deepqnetwork.py:176


@pytest.mark.parametrize("mode", MODES)
def test_forward_activations_layer_by_layer(mode):
    net, orc = _paired(4, mode)
    states = random_minibatch(32, 4, 8)[0]
    net.predict(states)
    _, acts = O.forward(orc.weights, states, keep=True)
    for name, dev in zip(("h1", "h2", "h3", "h4"), net.last_activations()):
        ref = acts[name]
        err = np.abs(dev - ref).max() / np.abs(ref).max()
        assert err <= 1e-4, (name, err)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("batch", [32, 1, 8, 40, 256])
def test_train_step_parity(mode, sched, batch):
    if mode == "fp32" and not (batch == 32 or (batch == 8 and sched == "serial")):
        pytest.skip("the SIMT twin is swept at batch 8 and 32 only (it is the cross-check, not the product)")
    net, orc = _paired(4, mode, batch=batch, stream=_stream(sched))
    costs = []
    net.callback = type("CB", (), {"on_train": staticmethod(lambda c: costs.append(c))})()
    mb = random_minibatch(batch, 4, 2)
    w0 = [w.copy() for w in orc.weights]
    net.train(mb, 0)
    ref_cost = orc.train(mb)
    preq, postq = net.last_q()
    scale = np.abs(orc.last["preq"]).max()
    assert np.abs(preq - orc.last["preq"]).max() <= 1e-3 * scale
    assert np.abs(postq - orc.last["postq"]).max() <= 1e-3 * np.abs(orc.last["postq"]).max()
    assert np.abs(net.last_deltas() - orc.last["deltas"]).max() <= 2e-3
    assert len(costs) == 1 and abs(costs[0] - ref_cost) <= 1e-3 * abs(ref_cost)
    for l, (g, r) in enumerate(zip(net.get_grads(), orc.last["grads"])):
        assert rel_l2(g, r) <= 2e-3, (l, rel_l2(g, r))
    ws, ss = net.get_weights()
    for l in range(5):
        assert rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l
        assert rel_l2(ss[l], orc.states[l]) <= 2e-3, l
    assert net.train_iterations == 1
    tw = net.get_weights(which=1, with_states=False)
    assert all((a == b).all() for a, b in zip(tw, w0))          # target untouched by train


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("sched", SCHEDS)
def test_rmsprop_bit_exact_given_same_gradient(mode, sched):
    """The optimizer arithmetic itself (Neon RMSProp order of operations) is bit-exact vs the
    oracle when fed the device's own gradient — in the generic k_optimizer (serial) and in the fused
    per-layer optimizers of the production schedule (k_opt_conv / k_opt_fc1)."""
    net, orc = _paired(4, mode, stream=_stream(sched))
    mb = random_minibatch(32, 4, 5)
    w0, s0 = net.get_weights()
    net.train(mb, 0)
    grads = net.get_grads()
    w1, s1 = net.get_weights()
    wr = [w.copy() for w in w0]
    sr = [s.copy() for s in s0]
    O.rmsprop_update(wr, sr, grads, 32)
    for l in range(5):
        assert (s1[l] == sr[l]).all(), l
        assert (w1[l] == wr[l]).all(), l


@pytest.mark.parametrize("mode", MODES)
def test_trajectory_20_steps_with_target_sync(mode):
    """k-step weight trajectory.  DQN + RMSProp is chaotic in fp32: elements whose second-moment
    state is dominated by the current gradient get a sign-like update of size lr/sqrt(1-decay), so
    a 1e-7 difference in a near-zero gradient becomes a full-size update difference.  Two
    *CPU* fp32 implementations of the same algorithm (numpy oracle vs torch-CPU) already diverge by
    ~0.3 rel-L2 of the update after 20 steps, so the 20-step criterion is calibrated live: the
    device must stay within 3x of how far the two CPU implementations drift apart; the first
    5 steps are held to an absolute 2e-2."""
    from oracle.dqn_torch import TorchDQN
    net, orc = _paired(6, mode, stream=_stream("branches"))
    tor = TorchDQN(orc.weights, orc.states)
    w0 = [w.copy() for w in orc.weights]
    ref_costs = []
    for i in range(20):
        mb = random_minibatch(32, 6, 100 + i, terminal_p=0.1)
        if i % 7 == 0:
            net.update_target_network()
            orc.update_target_network()
            tor.update_target_network()
        net.train(mb, 0)
        ref_costs.append(float(orc.train(mb)))
        tor.train(mb)
        if i == 4:
            ws = net.get_weights(with_states=False)
            for l in range(5):
                assert rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l
    ws = net.get_weights(with_states=False)
    for l in range(5):
        cpu_pair = rel_l2(tor.w[l].numpy() - w0[l], orc.weights[l] - w0[l])
        dev = rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l])
        assert dev <= 3 * cpu_pair + 2e-2, (l, dev, cpu_pair)
        assert rel_l2(ws[l], orc.weights[l]) <= 3e-2, l           # and the weights themselves stay close
    c = net.last_costs(20)
    assert c.shape == (20,) and np.isfinite(c).all()
    # per-step cost trace: tight while the trajectories coincide, bounded by the weight drift afterwards
    rel = np.abs(c - np.array(ref_costs)) / np.abs(ref_costs)
    assert rel[:5].max() <= 2e-3, rel[:5]
    assert rel.max() <= 5e-2, rel


@pytest.mark.parametrize("mode", MODES)
def test_fused_ring_training_equals_host_minibatch_training(mode):
    """agent.py:112-114 fused (sample -> frames read in place from the ring -> train) must do
    exactly what getMinibatch() + train(minibatch) does: same indexes, same weights."""
    from simple_dqn_b200 import ReplayMemory, Stream
    size, batch = 4000, 32
    orc_ring = ReplayOracle(size, batch_size=batch)
    synthetic_ring(orc_ring, seed=4, block=200, terminal_p=0.02)
    nets = []
    for fused in (True, False):
        # fused: non-default stream => CUDA-graph replay + side-stream branches;
        # unfused: legacy default stream => plain serial launches of the same kernels
        stream = Stream() if fused else None
        mem = ReplayMemory(size, make_args(), rng="device", stream=stream)
        mem.add_batch(orc_ring.actions, orc_ring.rewards, orc_ring.screens, orc_ring.terminals)
        mem.set_cursor(orc_ring.count, orc_ring.current)
        net, _ = _paired(4, mode, stream=stream)
        random.seed(77)
        mem.seed_device_rng(random)
        if fused:
            net.train_fused(mem, nsteps=2)
            net.train_fused(mem, nsteps=3)                      # second call replays the cached graph
        else:
            for _ in range(5):
                net.train(mem.getMinibatch(), 0)
        nets.append((net, mem))
    (nf, mf), (nu, mu) = nets
    assert (mf.read_device_rng() == mu.read_device_rng()).all()
    assert np.allclose(nf.last_costs(5), nu.last_costs(5), rtol=1e-6)
    for a, b in zip(nf.get_weights(with_states=False), nu.get_weights(with_states=False)):
        assert (a == b).all()                                   # same kernels, same data: bit-identical


@pytest.mark.parametrize("mode", MODES)
def test_device_minibatch_handle_and_statistics_pattern(mode):
    """statistics.py:83-90 pattern: unpack a minibatch, keep prestates, predict on them later."""
    from simple_dqn_b200 import DeviceMinibatch, ReplayMemory
    orc_ring = ReplayOracle(3000, batch_size=32)
    synthetic_ring(orc_ring, seed=6, block=100, terminal_p=0.02)
    mem = ReplayMemory(3000, make_args(), rng="python", device_minibatch=True)
    mem.add_batch(orc_ring.actions, orc_ring.rewards, orc_ring.screens, orc_ring.terminals)
    mem.set_cursor(orc_ring.count, orc_ring.current)
    net, orc = _paired(4, mode)
    random.seed(5)
    rng = MT19937.from_python(random)
    mb = mem.getMinibatch()
    assert isinstance(mb, DeviceMinibatch) and len(mb) == 5 and not mb.materialised
    net.train(mb, 0)                                            # trains in place from the ring
    ref_mb = orc_ring.getMinibatch(rng)
    orc.train(ref_mb)
    assert abs(net.last_costs(1)[0] - orc.last["cost"]) <= 1e-3 * abs(orc.last["cost"])
    prestates, actions, rewards, poststates, terminals = mem.getMinibatch()     # statistics.py:85
    ref = orc_ring.getMinibatch(rng)
    assert (prestates == ref[0]).all() and (actions == ref[1]).all() and (terminals == ref[4]).all()
    q = net.predict(prestates)                                  # statistics.py:90
    assert np.max(q, axis=1).shape == (32,)


@pytest.mark.parametrize("mode", MODES)
def test_state_buffer_predict_fast_path(mode):
    """agent.py:55-61: predict on the StateBuffer minibatch where only row 0 is live.  With no
    biases Q(all-zero state) == 0 exactly, so rows 1.. are returned as zeros."""
    from simple_dqn_b200 import StateBuffer
    net, orc = _paired(4, mode)
    buf = StateBuffer(make_args())
    rs = np.random.RandomState(0)
    for _ in range(6):
        buf.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    states = buf.getStateMinibatch()
    q = net.predict(states)
    ref = orc.predict(np.asarray(states))
    assert np.abs(q[0] - ref[0]).max() <= 1e-3 * np.abs(ref[0]).max()
    assert not q[1:].any() and not ref[1:].any()
    assert int(np.argmax(q[0])) == int(np.argmax(ref[0]))


def test_reference_flags_not_implemented_raise():
    from simple_dqn_b200 import DeepQNetwork
    for kw in (dict(batch_norm=True), dict(datatype="float16"), dict(stochastic_round=True),
               dict(screen_height=52, screen_width=40)):
        with pytest.raises(NotImplementedError):
            DeepQNetwork(4, make_args(**kw))
    with pytest.raises(AssertionError):                          # deepqnetwork.py:60-61
        DeepQNetwork(4, make_args(optimizer="sgd"))


def test_target_steps_zero_aliases_online():
    net = _net(4, "fp32", target_steps=0)
    mb = random_minibatch(32, 4, 9)
    net.train(mb, 0)
    a = net.get_weights(which=0, with_states=False)
    b = net.get_weights(which=1, with_states=False)
    assert all((x == y).all() for x, y in zip(a, b))            # deepqnetwork.py:72-73


@pytest.mark.parametrize("layout", ["pre-1.0", "neon-1.3.0"])
def test_snapshot_roundtrip(tmp_path, layout):
    net = _net(4, "fp32", random_seed=2)
    mb = random_minibatch(32, 4, 3)
    net.train(mb, 0)
    path = str(tmp_path / "w_1.prm")
    net.save_weights(path, layout=layout)
    d = pickle.load(open(path, "rb"))
    if layout == "pre-1.0":
        assert set(d) == {"epoch_index", "layer_params_states"} and len(d["layer_params_states"]) == 5
    else:
        assert len(d["model"]["config"]["layers"]) == 9
    net2 = _net(4, "fp32", random_seed=99)
    net2.load_weights(path)
    for (a, sa), (b, sb) in zip(zip(*net.get_weights()), zip(*net2.get_weights())):
        assert (a == b).all() and (sa == sb).all()
    states = mb[0]
    assert (net.predict(states) == net2.predict(states)).all()
    ws, ss = O.load_snapshot(path)                              # the oracle's reader agrees on the format
    assert all((a == b).all() for a, b in zip(ws, net.get_weights(with_states=False)))
