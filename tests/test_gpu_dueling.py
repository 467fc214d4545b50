"""The dueling network (b200dqn_net_config::dueling) on both engines and both schedules, each stage fed the device's own
inputs:
the advantages, V and Q of every network slot against tests/dueling_oracle.py rules 1 and 2 (slot 0 on the device's
H4, slots 1 and 2 on a dueling twin's H4 of the poststates), the deltas, row costs, TD errors and cost against their
restatement from the device's Q rows, dZ4 (and its fp16 planes) against rule 3, fc2's gradient against rule 4, and every
weight and optimizer
state plane after RMSProp, Adam and Adadelta against oracle.dqn_oracle's update of the device's gradient, all bit for
bit; the 1024-wide fc1 forward, dgrad and wgrad, and the convolutions behind them, inside test_gpu_kernels.py's float64
bounds.  Also: five fused steps against the numpy dueling step, fused against host-minibatch training, the predict
paths, checkpoints, target sync and the refusals."""
import os
import random

import numpy as np
import pytest

import dueling_oracle as D
import kernel_ref as K
import nstep_oracle as NS
from helpers import make_args
from oracle import dqn_oracle as O
from test_gpu_actions import _optimize_all, _ring, _ring_step
from test_gpu_distributional import _same_state
from test_gpu_flags import cost_finish, same
from test_gpu_kernels import _chain, _check, minibatch
from test_gpu_prioritized import _upload

pytestmark = pytest.mark.gpu

F32 = np.float32
ACTIONS = [1, 2, 4, 18, 32]
OPTIMIZERS = ["rmsprop", "adam", "adadelta"]
SCHEDS = ["branches", "serial"]
ENGINES = ["tcgen05", "fp32"]


def _stream(sched):
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


def make_net(A, batch, stream=None, double=False, optimizer="rmsprop", seed=3, mode="fp32", **kw):
    """A dueling net with Xavier weights, fc1 and fc2 x 3, small state in every optimizer plane, and (with a separate
    target network) a target perturbed away from the online one by 0.3 max|W| of noise per layer."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, random_seed=seed, double_dqn=double, optimizer=optimizer,
                                    dueling=True, **kw), math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    st = lambda w, scale: (np.abs(rs.randn(*w.shape)) * scale).astype(F32)
    states = {"rmsprop": lambda w: st(w, 1e-4),
              "adam": lambda w: [(rs.randn(*w.shape) * 1e-3).astype(F32), st(w, 1e-5)],
              "adadelta": lambda w: [st(w, 1e-5), st(w, 1e-9), (rs.randn(*w.shape) * 1e-4).astype(F32)]}[optimizer]
    net.set_weights(ws, [states(w) for w in ws])
    if kw.get("target_steps", 1):
        net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                        None, which=1)
    net.keep_grads(True)
    return net


def _twin_h4(net, weights, states):
    """H4 of `weights` on `states` from a dueling twin's predict: an independent source for slots 1 and 2."""
    from simple_dqn_b200 import DeepQNetwork
    twin = DeepQNetwork(net.num_actions, make_args(batch_size=net.batch_size, dueling=True), math_mode=net.math_mode)
    twin.set_weights(weights)
    twin.predict(states)
    return twin.last_activations()[3]


def check_step(net, train):
    """Run train() (one step; it returns the minibatch it trained on and its importance weights or None) and hold the
    step to the restatements.  Returns the minibatch."""
    A, rows = net.num_actions, net.batch_size
    w0, s0 = net.get_weights(with_states=False), net.get_states()
    tw = net.get_weights(which=1, with_states=False)
    mb, w = train()
    act = np.asarray(mb[1], np.int64)
    preq, postq = net.last_q()
    oq = net.last_online_postq() if net.double_dqn else None
    adv, val = net.last_advantages(), net.last_values()
    acts = net.last_activations()
    h4 = acts[3]
    assert h4.shape == (rows, 1024)
    # rules 1 and 2 on every slot
    slots = [(h4, w0[4])]
    slots.append((_twin_h4(net, tw, mb[3]), tw[4]))
    if oq is not None and any((x != y).any() for x, y in zip(w0, tw)):
        slots.append((_twin_h4(net, w0, mb[3]), w0[4]))
    elif oq is not None:                                      # target_steps = 0: slot 1 is the online net's forward
        assert (oq == postq).all()
    for z, (h, w5) in enumerate(slots):
        a_ref, v_ref = D.streams(h, w5)
        assert (adv[z] == a_ref).all() and (val[z] == v_ref).all(), z
        assert ((preq, postq, oq)[z] == D.aggregate(a_ref, v_ref)).all(), z
    # the TD step from the device's own Q rows
    d, rc, td = NS.head_restated(preq, postq, act, mb[2], mb[4], w=w, online_postq=oq)
    deltas = net.last_deltas()
    assert same(deltas, d), np.abs(deltas - d).max()
    assert same(net.last_row_costs(), rc)
    assert same(net.last_costs(1)[0], cost_finish(rc))
    if w is not None:
        assert same(net.last_td_errors(), td)
    # rules 3 and 4, then the update of every layer from the device's own gradient
    dA, dV = D.stream_grads(deltas[np.arange(rows), act], act, A)
    dz = net.last_dz()
    assert same(dz[3], D.dz4(h4, w0[4], dA, dV))
    if net.math_mode == "tcgen05":                            # the planes the tensor-core fc1 dgrad and wgrad read
        for got, ref in zip(net.last_dz4_planes(), K.split(dz[3])):
            assert (got.view(np.uint16) == ref.view(np.uint16)).all()
    grads = net.get_grads()
    assert same(grads[4], D.fc2_grad(h4, dA, dV))
    w1, s1 = net.get_weights(with_states=False), net.get_states()
    upd = [x.copy() for x in w0]
    _optimize_all(net.optimizer, upd, s0, grads, rows)
    for l in range(5):
        assert same(w1[l], upd[l]), l
        for k in range(net.num_states):
            assert same(s1[l][k], s0[l][k]), (l, k)
    if A == 1:
        assert (grads[4][0] == 0).all() and not np.signbit(grads[4][0]).any()
        if net.optimizer != "adam":                           # (Adam's momentum moves a weight without a gradient)
            assert same(w1[4][0], w0[4][0])                   # the advantage weights do not move
    # fc1 at 1024 units and the convolutions behind it within their float64 bounds
    h1, h2, h3, _ = acts
    dz1, dz2, dz3, dz4 = dz
    fc1_dgrad = lambda a, b: K.fc_dgrad(a, b).reshape(len(a), 64, 7, 7)
    e = net.math_mode
    c = lambda k: 1024 if k == "fc1_dgrad" else _chain(e, k, rows, 4)   # fc1_dgrad reduces over the 1024 units
    r = {}
    r.update(_check("fc1_fwd", e, K.fc_fwd, h3, w0[3], h4, c("fc1_fwd"), post=K.relu))
    r.update(_check("fc1_dgrad", e, fc1_dgrad, dz4, w0[3], dz3, c("fc1_dgrad"), mask=h3 > 0))
    r.update(_check("fc1_wgrad", e, K.fc_wgrad, h3, dz4, grads[3], c("fc1_wgrad")))
    r.update(_check("conv3_dgrad", e, K.conv_dgrad(2), dz3, w0[2], dz2, c("conv3_dgrad"), mask=h2 > 0))
    r.update(_check("conv3_wgrad", e, K.conv_wgrad(2), h2, dz3, grads[2], c("conv3_wgrad")))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, bad
    return mb


def _host_train(net, mb):
    def train():
        net.train(mb, 0)
        return mb, None
    return train


# ---------------------------------------------------------------------------------------------------- the step
@pytest.mark.parametrize("double", [False, True], ids=["vanilla", "double"])
@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("A", ACTIONS)
def test_dueling_step(A, mode, sched, double):
    """Batch 33 at every action count of the grid; the optimizer cycles with A."""
    net = make_net(A, 33, _stream(sched), double=double, optimizer=OPTIMIZERS[ACTIONS.index(A) % 3], mode=mode)
    check_step(net, _host_train(net, minibatch(33, 4, A, 40 + A)))


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("batch", [1, 32, 40, 256])
def test_dueling_step_batch_sizes(batch, mode, sched):
    net = make_net(4, batch, _stream(sched), double=batch == 40, optimizer=OPTIMIZERS[batch % 3], mode=mode)
    check_step(net, _host_train(net, minibatch(batch, 4, 4, 60 + batch)))


@pytest.mark.parametrize("double", [False, True], ids=["vanilla", "double"])
@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("mode", ENGINES)
def test_dueling_prioritized_nstep(mode, sched, double):
    """A = 32 from a prioritized ring with N = 3: k_head_duel<*, true>, importance-weighted deltas."""
    stream = _stream(sched)
    ring, mem = _ring(32, 33, stream, per=True, n=3, terminal_p=0.1)
    net = make_net(32, 33, stream, double=double, optimizer="adam", mode=mode)
    mb = check_step(net, lambda: (_ring_step(net, ring, mem, 3, 7), mem.last_weights))
    cut = mb[4].any(axis=1)
    assert len(np.unique(mem.last_weights)) > 1 and cut.any() and not cut.all()


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("mode", ENGINES)
def test_dueling_without_target_network(mode, sched):
    """target_steps = 0: the target network is the online one, and Double DQN's step is the vanilla step."""
    mb = minibatch(33, 4, 6, 5)
    nets = [make_net(6, 33, _stream(sched), double=d, target_steps=0, mode=mode) for d in (False, True)]
    for net in nets:
        check_step(net, _host_train(net, mb))
    _same_state(*nets)


@pytest.mark.parametrize("mode", ENGINES)
def test_double_tie_takes_the_first_index(mode):
    """The online net's advantage rows 5 and 27 are one non-negative row against small signed others: Q_online(s', 5)
    == Q_online(s', 27) is each row's maximum, exactly, and a* must be 5, as np.argmax."""
    net = make_net(32, 33, _stream("branches"), double=True, mode=mode)
    ws, ss = net.get_weights()
    col = np.abs(ws[4][5]) * F32(4)
    ws[4][:32] = ws[4][:32] * F32(0.01)
    ws[4][5] = ws[4][27] = col
    net.set_weights(ws, ss)
    mb = check_step(net, _host_train(net, minibatch(33, 4, 32, 9, terminal_p=0.0)))
    preq, postq = net.last_q()
    oq = net.last_online_postq()
    assert (oq[:, 5] == oq[:, 27]).all() and (oq[:, 5] == oq.max(axis=1)).all()
    assert (postq[:, 5] != postq[:, 27]).all()
    wrong = oq.copy()
    wrong[:, 27] = np.nextafter(wrong[:, 27], F32(np.inf))
    _, rc_wrong, _ = NS.head_restated(preq, postq, np.asarray(mb[1], np.int64), mb[2], mb[4], online_postq=wrong)
    assert (rc_wrong != net.last_row_costs()).any()


# ---------------------------------------------------------------------------------------------------- trajectories
@pytest.mark.parametrize("mode", ENGINES)
def test_fused_steps_track_the_numpy_step(mode):
    """Five fused steps from a ring (device MT19937 draw, RMSProp) within the trajectory bars of the numpy dueling
    step on the same minibatches."""
    from oracle.mt19937 import MT19937
    from oracle.replay_oracle import ReplayOracle, synthetic_ring
    from simple_dqn_b200 import ReplayMemory
    args = make_args(batch_size=32, random_seed=3, dueling=True)
    ring = ReplayOracle(2000, batch_size=32)
    synthetic_ring(ring, seed=1, block=100, terminal_p=0.01)
    mem = ReplayMemory(2000, args, rng="device")
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(4, args, math_mode=mode)
    ws, ss = net.get_weights()
    ws[3] *= F32(3)
    ws[4] *= F32(3)
    net.set_weights(ws, ss)
    net.update_target_network()
    w_np, s_np = [w.copy() for w in ws], [s.copy() for s in ss]
    random.seed(11)
    rng = MT19937.from_python(random)
    mem.seed_device_rng(random)
    net.train_fused(mem, nsteps=5)
    costs = [D.numpy_step(w_np, s_np, ws, ring.getMinibatch(rng))[0] for _ in range(5)]
    got = net.last_costs(5)
    assert np.allclose(got, costs, rtol=1e-3, atol=0), (got, costs)
    w1 = net.get_weights(with_states=False)
    for l in range(5):
        assert np.linalg.norm(w1[l] - w_np[l]) <= 2e-2 * np.linalg.norm(w_np[l] - ws[l]), l


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("mode", ENGINES)
def test_ring_and_host_minibatch_agree(mode, sched):
    """A step from the ring (frames read in place) and the same minibatch handed over from the host end in the same
    weights and state, bit for bit."""
    stream = _stream(sched)
    ring, mem = _ring(18, 32, stream)
    a, b = (make_net(18, 32, stream, optimizer="adam", mode=mode) for _ in range(2))
    mb = _ring_step(a, ring, mem, 1, 5)
    b.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]), 0)
    _same_state(a, b)
    assert same(a.last_advantages(), b.last_advantages()) and same(a.last_values(), b.last_values())


# ---------------------------------------------------------------------------------------------------- predict
@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("A,batch,live_rows", [(32, 32, (30, 31, 30, 29)), (1, 1024, (960, 961, 960, 959))])
def test_predict_paths(A, batch, live_rows, mode):
    """b200dqn_net_predict_device_host on both sides of the 960-float host-mapped capacity: live rows equal host
    predict bit for bit (and rule 2 on the device's H4), padding rows are +0 although a train step left non-zero Q."""
    import ctypes as C

    from simple_dqn_b200 import Stream
    from simple_dqn_b200 import _lib as L
    stream = Stream()
    net = make_net(A, batch, stream, mode=mode)
    net.train(minibatch(batch, 4, A, 3), 0)
    assert (net.last_q()[0] != 0).any()
    ring, mem = _ring(A, batch, stream)
    states = np.random.RandomState(A + batch).randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    _upload(mem, L.PTR_PRESTATES, states)
    ptr = C.c_void_p(mem.device_view(L.PTR_PRESTATES, np.uint8, states.shape).ptr)
    got = []
    for rows in live_rows:
        q = np.full((batch, A), np.nan, F32)
        L.call("b200dqn_net_predict_device_host", net._h, ptr, rows, L.np_ptr(q), net._stream)
        got.append((rows, q))
    host = net.predict(states)
    assert (host == D.q_rows(net.last_activations()[3], net.get_weights(with_states=False)[4])).all()
    for rows, q in got:
        assert (q[:rows] == host[:rows]).all(), rows
        assert same(q[rows:], np.zeros_like(q[rows:])), rows


# ---------------------------------------------------------------------------------------------------- weights
@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("A", [1, 18])
def test_checkpoints_sync_and_refusals(A, mode, tmp_path):
    """Shapes (1024, 3136) and (A + 1, 512); a trained net's weights and Adam state round-trip through both checkpoint
    layouts, and a loaded net's Q agrees with the numpy dueling forward; sync_target copies weights and state; a
    scalar checkpoint does not load into a dueling net, nor the reverse; comm_init is refused."""
    from simple_dqn_b200 import DeepQNetwork
    net = make_net(A, 32, optimizer="adam", mode=mode)
    assert net.dueling and net.layer_shapes()[3:] == [(1024, 3136), (A + 1, 512)]
    net.train(minibatch(32, 4, A, 5), 0)
    states = minibatch(32, 4, A, 6)[0]
    for layout in ("neon-1.3.0", "pre-1.0"):
        path = os.path.join(str(tmp_path), "w-%s.pkl" % layout)
        net.save_weights(path, layout=layout)
        other = make_net(A, 32, optimizer="adam", seed=9, mode=mode)
        other.load_weights(path)
        _same_state(net, other)
        ref = D.forward(other.get_weights(with_states=False), states)
        assert np.abs(other.predict(states) - ref).max() <= 1e-3 * np.abs(ref).max()
        scalar = DeepQNetwork(A, make_args(batch_size=32, optimizer="adam"), math_mode=mode)
        with pytest.raises(AssertionError, match="layer 3"):
            scalar.load_weights(path)
        spath = os.path.join(str(tmp_path), "s-%s.pkl" % layout)
        scalar.save_weights(spath, layout=layout)
        with pytest.raises(AssertionError, match="layer 3"):
            other.load_weights(spath)
    net.update_target_network()
    (w, s), t = net.get_weights(), net.get_weights(which=1)
    for l in range(5):
        assert same(t[0][l], w[l]) and same(t[1][l], s[l])
    with pytest.raises(NotImplementedError, match="dueling"):
        net.comm_init(bytes(128), 0, 2)
    with pytest.raises(AssertionError, match="dueling"):
        scalar.last_values()
