"""The scalar value head at every number of actions from 1 to 32 (kMaxActions), each stage fed the device's own inputs
as in test_gpu_distributional.py: the Q rows of every network slot against tests/head_oracle.py rule 1 (slot 0 on the
device's H4, slots 1 and 2 on a scalar twin's H4 of the poststates), the deltas, row costs, TD errors and cost against
their restatement from the device's Q rows, fc2's gradient (get_grads()[4]) against rule 2, and every weight and
optimizer state plane after RMSProp, Adam and Adadelta against oracle.dqn_oracle's update of the device's gradient, all
bit for bit; every other kernel of the step inside test_gpu_kernels.py's float64 bounds.

Also: ties in the Double DQN action choice (scalar and C51 heads) take the first index, as np.argmax; the predict
paths on either side of the host-mapped fast path's 960-float capacity; weights and checkpoints at odd action counts;
and the range of actions a step accepts."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import c51_oracle as C51
import head_oracle as H
import nstep_oracle as NS
from helpers import make_args
from oracle import dqn_oracle as O
from test_gpu_distributional import _check_train_step, _dnet, _ring_pair, _same_state, _slot_h4, _state
from test_gpu_flags import cost_finish, same
from test_gpu_kernels import backward_ratios, forward_ratios, minibatch
from test_gpu_prioritized import _upload

pytestmark = pytest.mark.gpu

F32 = np.float32
ACTIONS = [1, 2, 3, 5, 7, 8, 16, 17, 31, 32]
OPTIMIZERS = ["rmsprop", "adam", "adadelta"]
ENGINES = [("tcgen05", "branches"), ("tcgen05", "serial"), ("fp32", "branches"), ("fp32", "serial")]


def _L():
    from simple_dqn_b200 import _lib as L
    return L


def _stream(sched):
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


def make_net(A, mode, batch, stream=None, double=False, optimizer="rmsprop", seed=3):
    """Xavier weights with fc1 and fc2 x 3 (Q of order 1), small state in every optimizer plane, and a target network
    perturbed away from the online one (by 0.3 max|W| of noise per layer) so that the two prefer different actions."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, random_seed=seed, double_dqn=double, optimizer=optimizer),
                       math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    st = lambda w, scale: (np.abs(rs.randn(*w.shape)) * scale).astype(F32)
    states = {"rmsprop": lambda w: st(w, 1e-4),
              "adam": lambda w: [(rs.randn(*w.shape) * 1e-3).astype(F32), st(w, 1e-5)],
              "adadelta": lambda w: [st(w, 1e-5), st(w, 1e-9), (rs.randn(*w.shape) * 1e-4).astype(F32)]}[optimizer]
    net.set_weights(ws, [states(w) for w in ws])
    net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                    None, which=1)
    net.keep_grads(True)
    return net


def _ring(A, batch, stream, per=False, n=1, terminal_p=0.05):
    """A 3000-slot ring whose actions are drawn from 0..A-1, on the device and as a ReplayOracle; prioritized: stored
    priorities spanning four decades, so that the importance weights differ from 1."""
    ring, mem = _ring_pair(batch=batch, stream=stream, prioritized_replay=per, beta0=0.4, terminal_p=terminal_p)
    ring.actions[:] = np.random.RandomState(A).randint(0, A, len(ring.actions))
    _upload(mem, _L().PTR_ACTIONS, ring.actions)
    if per:
        _upload(mem, _L().PTR_PRIORITIES, np.random.default_rng(A).random(3000) ** 4 + 1e-3)
        mem.set_cursor(ring.count, ring.current)        # rebuilds every node of the tree over the new leaves
    mem.set_n_step(n)
    return ring, mem


def _ring_step(net, ring, mem, n, seed):
    """Train one step from the ring on drawn indexes; returns the gathered (batch, N) minibatch."""
    from simple_dqn_b200 import DeviceMinibatch
    idx = np.array(random.Random(seed).sample(range(4, 3000 - n + 1), net.batch_size), np.int32)
    mem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    return NS.gather(ring, idx.astype(np.int64), n)


def _optimize_all(optimizer, w0, s0, grads, rows, t=1):
    """oracle.dqn_oracle's update of every layer, in place on w0 / s0."""
    if optimizer == "rmsprop":
        O.rmsprop_update(w0, [s[0] for s in s0], grads, rows)
    elif optimizer == "adam":
        O.adam_update(w0, s0, grads, rows, t)
    else:
        O.adadelta_update(w0, s0, grads, rows)


def check_step(net, train):
    """Run train() (one step; it returns the minibatch it trained on and its importance weights or None) and hold the
    step to the restatements.  Returns the minibatch."""
    A = net.num_actions
    w0, s0 = net.get_weights(with_states=False), net.get_states()
    tw = net.get_weights(which=1, with_states=False)
    mb, w = train()
    act = np.asarray(mb[1], np.int64)
    preq, postq = net.last_q()
    oq = net.last_online_postq() if net.double_dqn else None
    acts = net.last_activations()
    h4 = acts[3]
    # rule 1 on every slot: slot 0 on the device's H4, slots 1 and 2 on a scalar twin's H4 of the poststates
    assert (preq == H.q_rows(h4, w0[4])).all()
    assert (postq == H.q_rows(_slot_h4(net, tw, mb[3]), tw[4])).all()
    if oq is not None:
        assert (oq == H.q_rows(_slot_h4(net, w0, mb[3]), w0[4])).all()
    # the TD step from the device's own Q rows
    d, rc, td = NS.head_restated(preq, postq, act, mb[2], mb[4], w=w, online_postq=oq)
    deltas = net.last_deltas()
    assert same(deltas, d), np.abs(deltas - d).max()
    assert same(net.last_row_costs(), rc)
    assert same(net.last_costs(1)[0], cost_finish(rc))
    if w is not None:
        assert same(net.last_td_errors(), td)
    # rule 2, then the update of every layer from the device's own gradient
    dz = net.last_dz()
    grads = net.get_grads()
    assert (grads[4] == H.fc2_grad(h4, deltas[np.arange(len(act)), act], act, A)).all()
    w1, s1 = net.get_weights(with_states=False), net.get_states()
    upd = [w.copy() for w in w0]
    _optimize_all(net.optimizer, upd, s0, grads, len(act))
    for l in range(5):
        assert same(w1[l], upd[l]), l
        for k in range(net.num_states):
            assert same(s1[l][k], s0[l][k]), (l, k)
    # every other kernel within its float64 bound (and dZ4 = delta W5 under the H4 mask, bit for bit)
    r = forward_ratios(net.math_mode, mb[0], w0, acts, preq)
    r.update(backward_ratios(net.math_mode, mb[0], w0, acts, dz, grads, deltas))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, bad
    return mb


def _host_train(net, mb):
    def train():
        net.train(mb, 0)
        return mb, None
    return train


# ---------------------------------------------------------------------------------------------------- action counts
@pytest.mark.parametrize("double", [False, True], ids=["vanilla", "double"])
@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("A", ACTIONS)
def test_action_count_sweep(A, mode, sched, double):
    """Batch 33 at every action count of the grid; the optimizer cycles with A, so that every engine, schedule and
    target sees all three."""
    opt = OPTIMIZERS[ACTIONS.index(A) % 3]
    net = make_net(A, mode, 33, _stream(sched), double=double, optimizer=opt)
    check_step(net, _host_train(net, minibatch(33, 4, A, 40 + A)))


@pytest.mark.parametrize("mode,sched", [("tcgen05", "branches"), ("fp32", "serial")])
@pytest.mark.parametrize("batch", [1, 257])
@pytest.mark.parametrize("A", [1, 17, 32])
def test_action_counts_at_batch_edges(A, batch, mode, sched):
    """One row (each 8-lane partial sum holds at most one term) and 257 rows (four fc1 splits, a ragged last lane)."""
    net = make_net(A, mode, batch, _stream(sched), double=A == 32, optimizer=OPTIMIZERS[A % 3])
    check_step(net, _host_train(net, minibatch(batch, 4, A, 60 + A)))


@pytest.mark.parametrize("double", [False, True], ids=["vanilla", "double"])
@pytest.mark.parametrize("mode,sched", ENGINES)
def test_max_actions_prioritized_nstep(mode, sched, double):
    """A = 32 from a prioritized ring with N = 3: the k_head<*, true> instantiations, importance-weighted deltas."""
    stream = _stream(sched)
    ring, mem = _ring(32, 33, stream, per=True, n=3, terminal_p=0.1)
    net = make_net(32, mode, 33, stream, double=double, optimizer="adam")

    def train():
        return _ring_step(net, ring, mem, 3, 7), mem.last_weights
    mb = check_step(net, train)
    cut = mb[4].any(axis=1)
    assert len(np.unique(mem.last_weights)) > 1 and cut.any() and not cut.all()


# ---------------------------------------------------------------------------------------------------- ties
TIE_RINGS = [(1, False), (1, True), (3, False), (3, True)]   # (N, prioritized)
TIES = {"pair": (5, 27), "all": (0, 31)}   # (j, k): the first maximum and the last one


def _tie_live_rows(mb):
    """Rows whose target reads Q of the poststate: no terminal in the window."""
    return ~np.asarray(mb[4]).reshape(len(mb[1]), -1).any(axis=1)


@pytest.mark.parametrize("case", sorted(TIES))
@pytest.mark.parametrize("n,per", TIE_RINGS)
@pytest.mark.parametrize("mode,sched", ENGINES)
def test_double_tie_takes_the_first_index(mode, sched, n, per, case):
    """The online net's fc2 columns j and k (pair), or all 32 (all), are one non-negative column, against small signed
    others: Q_online(s', j) == Q_online(s', k) is each row's maximum, exactly.  The target's columns stay distinct, so
    picking k instead of j would change the target.  a* must be j, as np.argmax."""
    j, k = TIES[case]
    stream = _stream(sched)
    ring, mem = _ring(32, 33, stream, per=per, n=n)
    net = make_net(32, mode, 33, stream, double=True)
    ws, ss = net.get_weights()
    col = np.abs(ws[4][j]) * F32(4)
    ws[4] = ws[4] * F32(0.01)
    if case == "pair":
        ws[4][j] = ws[4][k] = col
    else:
        ws[4][:] = col
    net.set_weights(ws, ss)

    def train():
        return _ring_step(net, ring, mem, n, 11), mem.last_weights if per else None
    mb = check_step(net, train)
    preq, postq = net.last_q()
    oq = net.last_online_postq()
    live = _tie_live_rows(mb)
    assert live.sum() >= 20
    assert (oq[:, j] == oq[:, k]).all() and (oq[:, j] == oq.max(axis=1)).all() and (np.argmax(oq, axis=1) == j).all()
    if case == "all":
        assert (oq == oq[:, :1]).all()
    assert (postq[live, j] != postq[live, k]).all()        # the choice decides the target on every live row
    w = mem.last_weights if per else None
    wrong = oq.copy()
    wrong[:, k] = np.nextafter(wrong[:, k], F32(np.inf))   # the restatement with a* = k: some row cost differs
    _, rc_wrong, _ = NS.head_restated(preq, postq, np.asarray(mb[1], np.int64), mb[2], mb[4], w=w, online_postq=wrong)
    assert (rc_wrong != net.last_row_costs())[live].any()


def _c51_tie_weights(ws, K, j, k, case):
    """Online fc2 blocks: j and k (pair) or every block (all) one block whose logits rise with the atom index, so its
    distribution sits near v_max; the others small and signed, so theirs is near uniform (Q near the support's mean)."""
    w5 = ws[4] * F32(0.01)
    ramp = (np.arange(K, dtype=np.float64) / K)[:, None]
    block = (np.abs(ws[4][j * K:(j + 1) * K]).astype(np.float64) * ramp).astype(F32)
    for a in ((j, k) if case == "pair" else range(len(w5) // K)):
        w5[a * K:(a + 1) * K] = block
    ws[4] = w5


@pytest.mark.parametrize("case", sorted(TIES))
@pytest.mark.parametrize("n,per", TIE_RINGS)
@pytest.mark.parametrize("mode,sched", ENGINES)
def test_c51_double_tie_takes_the_first_index(mode, sched, n, per, case):
    """The same with duplicated online action blocks and distinct target blocks: the projected target is the target
    network's distribution of block j (tests/c51_oracle.py rule 5 with the first index)."""
    from simple_dqn_b200 import DeviceMinibatch
    j, k = TIES[case]
    A, K = 32, 51
    stream = _stream(sched)
    ring, mem = _ring(A, 33, stream, per=per, n=n)
    net = _dnet(mode, A=A, atoms=K, batch=33, stream=stream, double=True)
    ws, ss = net.get_weights()
    _c51_tie_weights(ws, K, j, k, case)
    net.set_weights(ws, ss)
    before = _state(net)
    idx = np.array(random.Random(13).sample(range(4, 3000 - n + 1), 33), np.int32)
    mem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    mb = NS.gather(ring, idx.astype(np.int64), n)
    _check_train_step(net, before, mb[1].astype(np.int64), mb[2], mb[4], mb[3], w=mem.last_weights if per else None,
                      td=per)
    oq = net.last_online_postq()
    live = _tie_live_rows(mb)
    assert live.sum() >= 20
    assert (oq[:, j] == oq[:, k]).all() and (oq[:, j] == oq.max(axis=1)).all() and (np.argmax(oq, axis=1) == j).all()
    probs = net.last_distributions()
    assert (probs[2][:, j] == probs[2][:, k]).all()
    assert (probs[1][live, j] != probs[1][live, k]).any(axis=-1).all()    # distinct target blocks on every live row
    z, _, dz = C51.support(K, net.v_min, net.v_max)
    returns = [C51.n_step_return(mb[2][i], mb[4][i], 0.99) for i in range(33)]
    swapped = probs.copy()                                   # the restatement with a* = k: some target row differs
    swapped[1][:, j], swapped[1][:, k] = probs[1][:, k], probs[1][:, j]
    _, m_wrong, _ = C51.head(swapped, mb[1].astype(np.int64), returns, z, net.v_min, net.v_max, dz, double=True)
    assert (m_wrong != net.last_target_distribution())[live].any()


# ---------------------------------------------------------------------------------------------------- predict paths
PREDICT = {  # name: (A, batch, live row counts in call order, distributional)
    "A32": (32, 32, (30, 31, 30, 29), False),            # 960 floats (fast path), 992 (copy path), fast again
    "A1-b1024": (1, 1024, (960, 961, 960, 959), False),
    "c51-A32": (32, 32, (30, 31, 30, 29), True),
}


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("case", sorted(PREDICT))
def test_predict_paths_around_the_mapped_capacity(case, mode):
    """b200dqn_net_predict_device_host on device-resident states at live_rows * A on both sides of the 960 floats the
    host-mapped block holds: the captured fast path, the copy path, the fast path again (same rows: the graph is
    replayed) and at one row less (the graph is captured anew).  Live rows equal host predict bit for bit; padding rows
    are +0, also where a train step left non-zero Q in the device's buffer.  Then b200dqn_net_predict_device into a
    caller's buffer that holds non-zero values, at the same row counts."""
    from simple_dqn_b200 import Stream
    A, batch, live_rows, dist = PREDICT[case]
    L = _L()
    stream = Stream()
    net = _dnet(mode, A=A, batch=batch, stream=stream) if dist else make_net(A, mode, batch, stream)
    net.train(minibatch(batch, 4, A, 3), 0)                   # every row of the Q buffer now holds a train step's Q
    assert (net.last_q()[0] != 0).all(axis=1).any()
    ring, mem = _ring(A, batch, stream)
    states = np.random.RandomState(A + batch).randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    _upload(mem, L.PTR_PRESTATES, states)
    ptr = C.c_void_p(mem.device_view(L.PTR_PRESTATES, np.uint8, states.shape).ptr)
    got = []
    for rows in live_rows:
        q = np.full((batch, A), np.nan, F32)
        L.call("b200dqn_net_predict_device_host", net._h, ptr, rows, L.np_ptr(q), net._stream)
        got.append((rows, q))
    caller = net.device_view(L.NET_PTR_Q_TARGET, (batch, A)).ptr     # a device buffer of (batch, A) floats
    fill = np.full((batch, A), 7.0, F32)
    for rows in live_rows:
        L.call("b200dqn_copy_to_device", net.device, C.c_void_p(caller), L.np_ptr(fill), fill.nbytes, net._stream)
        L.call("b200dqn_net_predict_device", net._h, ptr, rows, C.c_void_p(caller), net._stream)
        got.append((rows, net._read_f32(L.NET_PTR_Q_TARGET, (batch, A))))
    host = net.predict(states)
    assert (host != 0).any(axis=1).all()
    for rows, q in got:
        assert (q[:rows] == host[:rows]).all(), rows
        assert same(q[rows:], np.zeros_like(q[rows:])), rows


# ---------------------------------------------------------------------------------------------------- weights
@pytest.mark.parametrize("A", [1, 2, 17, 32])
def test_weights_and_checkpoints_at_odd_action_counts(A, tmp_path):
    """fc2's Neon <-> internal conversion: a W5 of distinct entries comes back unchanged from either network; a trained
    net's weights and Adam state round-trip through both checkpoint layouts; a loaded net's Q agrees with the numpy
    oracle on what the file holds."""
    net = make_net(A, "tcgen05", 32, optimizer="adam")
    for which in (0, 1):
        ws = net.get_weights(which=which, with_states=False)
        perm = np.random.RandomState(A + which).permutation(A * 512).reshape(A, 512)
        ws[4] = ((perm + 1) * np.where(perm % 3 == 0, -1, 1) * 2.0 ** -14).astype(F32)
        assert len(np.unique(ws[4])) == A * 512
        net.set_weights(ws, None, which=which)
        for a, b in zip(net.get_weights(which=which, with_states=False), ws):
            assert same(a, b)
    net.train(minibatch(32, 4, A, 5), 0)
    states = minibatch(32, 4, A, 6)[0]
    for layout in ("neon-1.3.0", "pre-1.0"):
        path = os.path.join(str(tmp_path), "w-%s.pkl" % layout)
        net.save_weights(path, layout=layout)
        other = make_net(A, "tcgen05", 32, optimizer="adam", seed=9)
        other.load_weights(path)
        _same_state(net, other)
        ref = O.forward(other.get_weights(with_states=False), states)
        assert np.abs(other.predict(states) - ref).max() <= 1e-3 * np.abs(ref).max()


# ---------------------------------------------------------------------------------------------------- action range
@pytest.mark.parametrize("A", [1, 32])
def test_action_range(A):
    """Action A - 1 trains (its column of the deltas is the only non-zero one); actions A and 255 are refused: a host
    minibatch before anything runs, a ring step through the sticky flag its head raises (the head clamps the action,
    so nothing reads out of bounds) at the next read of the costs."""
    from simple_dqn_b200 import DeepQNetwork, DeviceMinibatch, Stream
    for bad in (0, 33):
        with pytest.raises(AssertionError, match="num_actions"):
            DeepQNetwork(bad, make_args(), math_mode="tcgen05")
    net = make_net(A, "tcgen05", 8)
    mb = list(minibatch(8, 4, A, 1, terminal_p=0.0))
    mb[1] = np.full(8, A - 1, np.uint8)
    net.train(tuple(mb), 0)
    assert (net.last_deltas()[:, A - 1] != 0).all() and not net.last_deltas()[:, :A - 1].any()
    for bad in (A, 255):
        wrong = list(mb)
        wrong[1] = mb[1].copy()
        wrong[1][5] = bad
        with pytest.raises(AssertionError):
            net.train(tuple(wrong), 0)
    assert np.isfinite(net.last_costs(1)).all()               # the refused minibatches left the net usable
    for bad in (None, A, 255):
        stream = Stream()
        ring, mem = _ring(A, 8, stream)
        ring.actions[:] = A - 1
        if bad is not None:
            ring.actions[40] = bad
        _upload(mem, _L().PTR_ACTIONS, ring.actions)
        net = make_net(A, "tcgen05", 8, stream)
        mem.set_indexes(np.array([10, 20, 30, 40, 50, 60, 70, 80], np.int32))
        net.train(DeviceMinibatch(mem, sampled=True))
        if bad is None:
            assert np.isfinite(net.last_costs(1)).all()
            assert (net.last_deltas()[:, A - 1] != 0).any() and not net.last_deltas()[:, :A - 1].any()
        else:
            with pytest.raises(AssertionError, match="num_actions"):
                net.last_costs(1)
