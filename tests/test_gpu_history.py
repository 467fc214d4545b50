"""--history_length other than 4 on both network engines (main.py:34; deepqnetwork.py:37 takes the H frames of a
state as conv1's input channels).  conv1 has 64*H filter rows, one 64-tap k-block per frame; every later layer
keeps its shape.  Bars as in tests/test_gpu_net.py.

H runs over 1, 2, 3, 5 and 8: odd and even, below, at and above the tensor-core engine's 4-stage operand ring, and an
odd number of 64-row m chunks in conv1's weight gradient.  H = 16, the largest implemented, is in the predict and
train-step sweeps."""
import pickle
import random

import numpy as np
import pytest

from helpers import make_args, rel_l2
from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tcgen05"]
SCHEDS = ["serial", "branches"]
HISTS = [1, 2, 3, 5, 8]


def _minibatch(n, hist, num_actions, seed, terminal_p=0.3):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8)
    return (pre, rs.randint(0, num_actions, n).astype(np.uint8), rs.randint(-3, 4, n).astype(np.int64), post,
            rs.rand(n) < terminal_p)


def _stream(sched):
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


def _net(hist, mode, stream=None, **kw):
    from simple_dqn_b200 import DeepQNetwork
    return DeepQNetwork(4, make_args(history_length=hist, **kw), math_mode=mode, stream=stream)


def _paired(hist, mode, seed=3, batch=32, stream=None):
    """A device net and an oracle net holding identical fp32 weights (trained-looking scale)."""
    net = _net(hist, mode, stream=stream, batch_size=batch, random_seed=seed)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * np.float32(3.0)
    ws[4] = ws[4] * np.float32(3.0)
    rs = np.random.RandomState(seed)
    ss = [np.abs(rs.randn(*w.shape)).astype(np.float32) * np.float32(1e-4) for w in ws]
    net.set_weights(ws, ss)
    net.update_target_network()
    net.keep_grads(True)
    orc = O.DQNOracle(4, batch_size=batch, weights=ws, states=ss)
    return net, orc


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hist", HISTS + [16])
def test_xavier_init_matches_oracle_draw_order(mode, hist):
    net = _net(hist, mode, random_seed=11)
    ws, ss = net.get_weights()
    ref = O.xavier_init(4, seed=11, history_length=hist)
    assert ws[0].shape == (64 * hist, 32)
    assert [w.shape for w in ws] == O.layer_shapes(4, history_length=hist)
    assert all((a == b).all() for a, b in zip(ws, ref))
    assert all(not s.any() for s in ss)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hist", HISTS + [16])
@pytest.mark.parametrize("batch", [32, 1, 40])
def test_predict_parity(mode, hist, batch):
    net, orc = _paired(hist, mode, batch=batch)
    states = _minibatch(batch, hist, 4, 1)[0]
    q = net.predict(states)
    ref = orc.predict(states)
    assert q.shape == (batch, 4) and q.dtype == np.float32
    assert np.abs(q - ref).max() <= 1e-3 * np.abs(ref).max(), np.abs(q - ref).max() / np.abs(ref).max()
    with pytest.raises(AssertionError):                        # a window of another history length (:176)
        net.predict(_minibatch(batch, hist + 1, 4, 1)[0])


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hist", HISTS)
def test_forward_activations_layer_by_layer(mode, hist):
    net, orc = _paired(hist, mode)
    states = _minibatch(32, hist, 4, 8)[0]
    net.predict(states)
    _, acts = O.forward(orc.weights, states, keep=True)
    for name, dev in zip(("h1", "h2", "h3", "h4"), net.last_activations()):
        ref = acts[name]
        err = np.abs(dev - ref).max() / np.abs(ref).max()
        assert err <= 1e-4, (name, err)


# the SIMT twin at batch 32; the tensor-core engine also at 1 (one partial M tile), 40 and 256
TRAIN_CASES = ([("fp32", h, 32) for h in HISTS + [16]] + [("tcgen05", h, b) for h in HISTS + [16] for b in (32, 1, 40)] +
               [("tcgen05", h, 256) for h in (1, 3, 8)])


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("mode,hist,batch", TRAIN_CASES)
def test_train_step_parity(mode, hist, batch, sched):
    net, orc = _paired(hist, mode, batch=batch, stream=_stream(sched))
    costs = []
    net.callback = type("CB", (), {"on_train": staticmethod(lambda c: costs.append(c))})()
    mb = _minibatch(batch, hist, 4, 2)
    w0 = [w.copy() for w in orc.weights]
    net.train(mb, 0)
    ref_cost = orc.train(mb)
    preq, postq = net.last_q()
    assert np.abs(preq - orc.last["preq"]).max() <= 1e-3 * np.abs(orc.last["preq"]).max()
    assert np.abs(postq - orc.last["postq"]).max() <= 1e-3 * np.abs(orc.last["postq"]).max()
    assert len(costs) == 1 and abs(costs[0] - ref_cost) <= 1e-3 * abs(ref_cost)
    grads = net.get_grads()
    assert grads[0].shape == (64 * hist, 32)
    for l, (g, r) in enumerate(zip(grads, orc.last["grads"])):
        assert rel_l2(g, r) <= 2e-3, (l, rel_l2(g, r))
    ws, ss = net.get_weights()
    for l in range(5):
        assert rel_l2(ws[l] - w0[l], orc.weights[l] - w0[l]) <= 2e-2, l
        assert rel_l2(ss[l], orc.states[l]) <= 2e-3, l
    tw = net.get_weights(which=1, with_states=False)
    assert all((a == b).all() for a, b in zip(tw, w0))          # target untouched by train


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("hist", HISTS)
def test_rmsprop_bit_exact_given_same_gradient(mode, sched, hist):
    """The fused conv1 optimizer (split-K reduction over 64*H rows, update, tile-image refresh) is bit-exact
    against the oracle's RMSProp fed the device's own gradient."""
    net, _ = _paired(hist, mode, stream=_stream(sched))
    mb = _minibatch(32, hist, 4, 5)
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
    # the refreshed conv1 tile image is what the next forward multiplies by
    states = _minibatch(32, hist, 4, 6)[0]
    q = net.predict(states)
    ref = O.forward(wr, states)
    assert np.abs(q - ref).max() <= 1e-3 * np.abs(ref).max()


def _ring(hist, seed, terminal_p):
    orc_ring = ReplayOracle(3000, history_length=hist, batch_size=32)
    synthetic_ring(orc_ring, seed=seed, block=150, terminal_p=terminal_p)
    return orc_ring


def _device_ring(orc_ring, hist, stream=None, **kw):
    from simple_dqn_b200 import ReplayMemory
    mem = ReplayMemory(orc_ring.size, make_args(history_length=hist), stream=stream, **kw)
    mem.add_batch(orc_ring.actions, orc_ring.rewards, orc_ring.screens, orc_ring.terminals)
    mem.set_cursor(orc_ring.count, orc_ring.current)
    return mem


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hist", HISTS)
def test_fused_ring_training_equals_host_minibatch_training(mode, hist):
    """train_fused reads the H-frame windows in place from the ring; getMinibatch() + train copies them out first.
    The ring is terminal-heavy so that many draws are rejected.  Indexes and gathered frames of the host path equal
    ReplayOracle's, and both paths end with bit-identical weights."""
    from simple_dqn_b200 import Stream
    orc_ring = _ring(hist, seed=4, terminal_p=0.1)
    nets = []
    for fused in (True, False):
        stream = Stream() if fused else None
        mem = _device_ring(orc_ring, hist, stream=stream, rng="device")
        net, _ = _paired(hist, mode, stream=stream)
        random.seed(77)
        rng = MT19937.from_python(random)
        mem.seed_device_rng(random)
        if fused:
            net.train_fused(mem, nsteps=2)
            net.train_fused(mem, nsteps=3)                      # the second call replays the cached graph
        else:
            for _ in range(5):
                mb = mem.getMinibatch()
                idx = orc_ring.sample_indexes(rng)
                ref = orc_ring.gather(idx)
                assert (mem.last_indexes == idx).all()
                for a, b in zip(mb, ref):
                    assert (np.asarray(a) == np.asarray(b)).all()
                net.train(mb, 0)
        nets.append((net, mem))
    (nf, mf), (nu, mu) = nets
    assert (mf.read_device_rng() == mu.read_device_rng()).all()
    assert np.allclose(nf.last_costs(5), nu.last_costs(5), rtol=1e-6)
    for a, b in zip(nf.get_weights(with_states=False), nu.get_weights(with_states=False)):
        assert (a == b).all()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hist", HISTS)
def test_device_minibatch_handle_and_statistics_pattern(mode, hist):
    from simple_dqn_b200 import DeviceMinibatch
    orc_ring = _ring(hist, seed=6, terminal_p=0.02)
    mem = _device_ring(orc_ring, hist, rng="python", device_minibatch=True)
    net, orc = _paired(hist, mode)
    random.seed(5)
    rng = MT19937.from_python(random)
    mb = mem.getMinibatch()
    assert isinstance(mb, DeviceMinibatch) and not mb.materialised
    net.train(mb, 0)                                            # trains in place from the ring
    orc.train(orc_ring.getMinibatch(rng))
    assert abs(net.last_costs(1)[0] - orc.last["cost"]) <= 1e-3 * abs(orc.last["cost"])
    prestates, actions, rewards, poststates, terminals = mem.getMinibatch()     # statistics.py:85
    ref = orc_ring.getMinibatch(rng)
    assert prestates.shape == (32, hist, 84, 84)
    assert (prestates == ref[0]).all() and (poststates == ref[3]).all() and (actions == ref[1]).all()
    q = net.predict(prestates)                                  # statistics.py:90
    qr = orc.predict(np.asarray(prestates))
    assert np.abs(q - qr).max() <= 1e-3 * np.abs(qr).max()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("hist", HISTS)
def test_state_buffer_predict_fast_path(mode, hist):
    from simple_dqn_b200 import StateBuffer
    net, orc = _paired(hist, mode)
    buf = StateBuffer(make_args(history_length=hist))
    rs = np.random.RandomState(0)
    for _ in range(hist + 2):
        buf.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    states = buf.getStateMinibatch()
    assert states.shape == (32, hist, 84, 84)
    q = net.predict(states)
    ref = orc.predict(np.asarray(states))
    assert np.abs(q[0] - ref[0]).max() <= 1e-3 * np.abs(ref[0]).max()
    assert not q[1:].any() and not ref[1:].any()
    other = StateBuffer(make_args(history_length=hist + 1))
    with pytest.raises(AssertionError):                          # a window of another history length
        net.predict(other.getStateMinibatch())


@pytest.mark.parametrize("layout", ["pre-1.0", "neon-1.3.0"])
@pytest.mark.parametrize("hist", HISTS)
def test_snapshot_roundtrip(tmp_path, layout, hist):
    net = _net(hist, "fp32", random_seed=2)
    mb = _minibatch(32, hist, 4, 3)
    net.train(mb, 0)
    path = str(tmp_path / "w_1.prm")
    net.save_weights(path, layout=layout)
    if layout == "neon-1.3.0":
        assert pickle.load(open(path, "rb"))["train_input_shape"] == (hist, 84, 84)
    net2 = _net(hist, "tcgen05", random_seed=99)
    net2.load_weights(path)
    for (a, sa), (b, sb) in zip(zip(*net.get_weights()), zip(*net2.get_weights())):
        assert (a == b).all() and (sa == sb).all()
    q, q2 = net.predict(mb[0]), net2.predict(mb[0])
    assert np.abs(q - q2).max() <= 1e-3 * np.abs(q).max()


@pytest.mark.parametrize("layout", ["pre-1.0", "neon-1.3.0"])
def test_checkpoint_of_another_history_length_is_rejected(tmp_path, layout):
    path = str(tmp_path / "w_4.prm")
    _net(4, "fp32", random_seed=2).save_weights(path, layout=layout)
    net = _net(2, "fp32", random_seed=3)
    w0 = net.get_weights(with_states=False)
    with pytest.raises(AssertionError):
        net.load_weights(path)
    assert all((a == b).all() for a, b in zip(w0, net.get_weights(with_states=False)))


@pytest.mark.parametrize("mode", MODES)
def test_history_length_out_of_range(mode):
    with pytest.raises(AssertionError):
        _net(0, mode)
    with pytest.raises(NotImplementedError, match="1..16"):
        _net(17, mode)


@pytest.mark.parametrize("mode", MODES)
def test_train_fused_with_ring_of_another_history_length(mode):
    orc_ring = _ring(3, seed=4, terminal_p=0.02)
    mem = _device_ring(orc_ring, 3, rng="device")
    net = _net(2, mode)
    with pytest.raises(AssertionError):
        net.train_fused(mem, 1)


@pytest.mark.parametrize("hist", [2, 8])
def test_comm_init_needs_four_frames(hist):
    net = _net(hist, "tcgen05")
    with pytest.raises(NotImplementedError, match="history_length"):
        net.comm_init(bytes(128), 0, 2)
