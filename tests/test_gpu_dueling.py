"""The dueling network (b200dqn_net_config::dueling) on both engines and both schedules, each stage fed the device's own
inputs:
the advantages, V and Q of every network slot against tests/dueling_oracle.py rules 1 and 2 (slot 0 on the device's
H4, slots 1 and 2 on a dueling twin's H4 of the poststates), the deltas, row costs, TD errors and cost against their
restatement from the device's Q rows, dZ4 (and its fp16 planes) against rule 3, fc2's gradient against rule 4, and every
weight and optimizer
state plane after RMSProp, Adam and Adadelta against oracle.dqn_oracle's update of the device's gradient, all bit for
bit; all eleven GEMM-shaped kernels (the convolutions and the 1024-wide fc1, forward, dgrad and wgrad) inside
test_gpu_kernels.py's float64 bounds, and after the update the forward kernels again, on the refreshed tile images.
That step runs across the batch-size dispatch (test_gpu_kernels.py's sweep: one or two conv2/conv3 forward kernels,
7 or 4 fc1 split-K partials summed by k_head_duel, 1 to 48 conv weight-gradient splits), at history lengths 1 to 16,
on the SIMT engine above 256 rows and under forced fc1 split counts.  Bit-for-bit identities: the optimizer-refreshed
tile images equal a fresh pack of the updated weights, the synced target network equals the online one, keep_grads
changes nothing, and Double DQN switched on in a live net equals Double DQN from creation.  Also: five fused steps
against the numpy dueling step, fused against host-minibatch training, the predict paths, checkpoints, target sync and
the refusals."""
import json
import os
import random
import subprocess
import sys

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
from test_gpu_kernels import SWEEP, _check, gemm_backward_ratios, gemm_forward_ratios, minibatch
from test_gpu_prioritized import _upload

pytestmark = pytest.mark.gpu

F32 = np.float32
ACTIONS = [1, 2, 4, 18, 32]
OPTIMIZERS = ["rmsprop", "adam", "adadelta"]
SCHEDS = ["branches", "serial"]
ENGINES = ["tcgen05", "fp32"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORST = {}          # kernel -> largest ratio of error to bound on the dueling steps and predicts of this module


def _note(ratios):
    for k, v in ratios.items():
        WORST[k] = max(WORST.get(k, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest |error| / bound per kernel on a dueling net:")
    for k in sorted(WORST):
        print("  %-20s %8.3g" % (k, WORST[k]))


def _stream(sched):
    from simple_dqn_b200 import Stream
    return Stream() if sched == "branches" else None


def make_net(A, batch, stream=None, double=False, optimizer="rmsprop", seed=3, mode="fp32", keep=True, **kw):
    """A dueling net with Xavier weights, fc1 and fc2 x 3, small state in every optimizer plane, and (with a separate
    target network) a target perturbed away from the online one by 0.3 max|W| of noise per layer.  keep: keep_grads,
    so that last_dz() has dZ1..dZ3."""
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
    net.keep_grads(keep)
    return net


def _twin_h4(net, weights, states):
    """H4 of `weights` on `states` from a dueling twin's predict: an independent source for slots 1 and 2."""
    from simple_dqn_b200 import DeepQNetwork
    twin = DeepQNetwork(net.num_actions, make_args(batch_size=net.batch_size, history_length=net.history_length,
                                                   dueling=True), math_mode=net.math_mode)
    twin.set_weights(weights)
    twin.predict(states)
    return twin.last_activations()[3]


def check_step(net, train, fc1_forced=0, updated=True):
    """Run train() (one step; it returns the minibatch it trained on and its importance weights or None) and hold the
    step to the restatements.  fc1_forced: the split count B200DQN_FC1_SPLITS forces in this process.  updated: then
    predict on fresh states and hold the forward kernels, which read the tile images the update refreshed, to their
    bounds on the updated weights (this overwrites the step's slot-0 Q, activations and advantages).  Returns the
    minibatch."""
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
    # every GEMM-shaped kernel (fc1 at 1024 units, the convolutions around it) within its float64 bound
    e = net.math_mode
    r = gemm_forward_ratios(e, mb[0], w0, acts, fc1_forced)
    r.update(gemm_backward_ratios(e, mb[0], w0, acts, dz, grads))
    if updated:     # the forward on the refreshed tile images; rules 1 and 2 on the device's H4 of the new weights
        fresh = minibatch(rows, net.history_length, A, 1234)[0]
        q = net.predict(fresh)
        acts1 = net.last_activations()
        r.update({k + "@updated": v for k, v in gemm_forward_ratios(e, fresh, w1, acts1, fc1_forced).items()})
        a_ref, v_ref = D.streams(acts1[3], w1[4])
        assert (net.last_advantages()[0] == a_ref).all() and (net.last_values()[0] == v_ref).all()
        assert (q == D.aggregate(a_ref, v_ref)).all()
    _note(r)
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
    mb = check_step(net, _host_train(net, minibatch(33, 4, 32, 9, terminal_p=0.0)), updated=False)
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


# ---------------------------------------------------------------------------------------------------- dispatch
# Each float64 check costs about 20 ms of host time per row, so the dispatch cases pair their switches instead of
# crossing them: every batch of the sweep runs once, the (schedule, Double DQN) pairs cycling with it, and each side
# of the 64/65 and 256/257 boundaries runs on both schedules.
_PAIRS = [("branches", False), ("serial", True), ("serial", False), ("branches", True)]
SWEEP_RUNS = [(b, *_PAIRS[i % 4]) for i, b in enumerate(SWEEP)] + [(257, "serial", False)]


@pytest.mark.parametrize("batch,sched,double", SWEEP_RUNS,
                         ids=["%d-%s-%s" % (b, s, "double" if d else "vanilla") for b, s, d in SWEEP_RUNS])
def test_dueling_step_kernels(batch, sched, double):
    """The tensor-core step across the batch-size dispatch (test_gpu_kernels.py's table): above 256 rows fc1_fwd writes
    4 split-K partials per slot and k_head_duel sums 4; the optimizer cycles with the batch."""
    net = make_net(4, batch, _stream(sched), double=double, optimizer=OPTIMIZERS[SWEEP.index(batch) % 3],
                   mode="tcgen05")
    check_step(net, _host_train(net, minibatch(batch, 4, 4, 70 + batch)))


def test_dueling_forward_kernels_at_4096():
    """Forward only, 4096 rows (4 fc1 splits, 32 M-tiles of samples): the 1024-wide fc1 within its bound, and A, V and
    Q from the device's own H4 bit for bit.  (The convolutions are the scalar net's kernels, which
    test_gpu_kernels.py holds at 4096 rows; their float64 references there take about 20 s of host time.)"""
    net = make_net(4, 4096, mode="tcgen05")
    states = minibatch(4096, 4, 4, 5)[0]
    q = net.predict(states)
    ws, acts = net.get_weights(with_states=False), net.last_activations()
    r = _check("fc1_fwd", "tcgen05", K.fc_fwd, acts[2], ws[3], acts[3], K.chain("fc1_fwd", 4096), post=K.relu)
    _note(r)
    assert all(v <= 1.0 for v in r.values()), r
    a_ref, v_ref = D.streams(acts[3], ws[4])
    assert (net.last_advantages()[0] == a_ref).all() and (net.last_values()[0] == v_ref).all()
    assert (q == D.aggregate(a_ref, v_ref)).all()


HIST_RUNS = [(b, h, (b + h) % 2 == 1) for h in (1, 5, 16) for b in (1, 64, 65)]


@pytest.mark.parametrize("batch,hist,double", HIST_RUNS,
                         ids=["%d-%d-%s" % (b, h, "double" if d else "vanilla") for b, h, d in HIST_RUNS])
def test_dueling_history_lengths(batch, hist, double):
    """conv1's K = 64·H on both sides of the one-kernel conv2/conv3 forward; the slot-1 and slot-2 twins run H too."""
    net = make_net(4, batch, _stream("branches"), double=double, optimizer=OPTIMIZERS[hist % 3], mode="tcgen05",
                   history_length=hist)
    check_step(net, _host_train(net, minibatch(batch, hist, 4, 80 + hist)))


@pytest.mark.parametrize("batch,double", [(65, True), (257, False)], ids=["65-double", "257-vanilla"])
def test_dueling_simt_engine_above_64_rows(batch, double):
    net = make_net(4, batch, double=double, optimizer="adam", mode="fp32")
    check_step(net, _host_train(net, minibatch(batch, 4, 4, 90 + batch)))


def _child_steps(splits):
    """check_step at batch 33 (vanilla) and 257 (Double DQN) in a child process (B200DQN_FC1_SPLITS is read once per
    process); returns the child's worst ratio per kernel."""
    code = ("import json, sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_dueling as T\n"
            "for batch, double in ((33, False), (257, True)):\n"
            "    net = T.make_net(4, batch, T._stream('branches'), double=double, mode='tcgen05')\n"
            "    T.check_step(net, T._host_train(net, T.minibatch(batch, 4, 4, 21)), fc1_forced=%d)\n"
            "print('RATIOS', json.dumps(T.WORST))\n" % (ROOT, os.path.join(ROOT, "tests"), splits))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=dict(os.environ, B200DQN_FC1_SPLITS=str(splits)),
                         capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("RATIOS ")][0]
    return json.loads(line[len("RATIOS "):])


@pytest.mark.parametrize("splits", [1, 4, 14])
def test_dueling_fc1_forced_splits(splits):
    """1, 4 and 14 split-K partials of 1024 units per slot; Double DQN at 14 fills the whole three-slot buffer."""
    r = _child_steps(splits)
    _note(r)
    assert {"fc1_fwd", "fc1_fwd@updated", "fc1_dgrad", "conv1_wgrad"} <= set(r)


# ---------------------------------------------------------------------------------------------------- identities
@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("opt,batch", [("rmsprop", 1), ("adam", 33), ("adadelta", 257)])
def test_tile_images_after_an_update(opt, batch, sched):
    """Two updates at lr 0.01 (the branches schedule refreshes the fc1 image inside k_opt_fc1<1024>, the serial one
    repacks it after the update): a twin loaded with the updated fp32 weights predicts the same Q, A, V and H1..H4,
    bit for bit.  A stale hi or lo plane of any layer's image would change them."""
    stream = _stream(sched)
    net = make_net(4, batch, stream, optimizer=opt, mode="tcgen05", learning_rate=0.01)
    for t in (1, 2):
        net.train(minibatch(batch, 4, 4, 100 + t), 0)
    twin = make_net(4, batch, stream, optimizer=opt, seed=8, mode="tcgen05")
    twin.set_weights(net.get_weights(with_states=False))
    states = minibatch(batch, 4, 4, 99)[0]
    assert same(net.predict(states), twin.predict(states))
    assert same(net.last_advantages()[0], twin.last_advantages()[0])
    assert same(net.last_values()[0], twin.last_values()[0])
    for a, b in zip(net.last_activations(), twin.last_activations()):
        assert same(a, b)


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("batch", [1, 33, 65, 256, 257])
def test_target_net_equals_online_net(batch, mode):
    """Freshly synced target, poststates = prestates: the target slot (the fc1 image the sync copied, 1024 units wide)
    gives postq == preq, and the same A and V, bit for bit."""
    net = make_net(4, batch, _stream("branches"), mode=mode)
    net.train(minibatch(batch, 4, 4, 13), 0)      # the online images now differ from the ones the sync copies
    net.update_target_network()
    states = minibatch(batch, 4, 4, 14)[0]
    net.train(minibatch(batch, 4, 4, 15, states=states), 0)
    preq, postq = net.last_q()
    assert (preq == postq).all()
    adv, val = net.last_advantages(), net.last_values()
    assert (adv[1] == adv[0]).all() and (val[1] == val[0]).all()


@pytest.mark.parametrize("sched,batch,double", [("branches", 32, False), ("serial", 32, True),
                                                ("branches", 257, True), ("serial", 257, False)],
                         ids=["branches-32-vanilla", "serial-32-double", "branches-257-double", "serial-257-vanilla"])
def test_keep_grads_changes_nothing(sched, batch, double):
    """keep_grads off (the production path: the dgrads write no fp32 dZ) and on end in the same weights, every
    optimizer state plane and the same gradients, bit for bit."""
    nets = [make_net(4, batch, _stream(sched), double=double, mode="tcgen05", keep=k) for k in (False, True)]
    mb = minibatch(batch, 4, 4, 17)
    for net in nets:
        for _ in range(2):
            net.train(mb, 0)
    _same_state(*nets)
    for a, b in zip(nets[0].get_grads(), nets[1].get_grads()):
        assert same(a, b)


@pytest.mark.parametrize("mode", ENGINES)
def test_double_switched_on_live_equals_switched_on_at_creation(mode):
    """test_gpu_double.py's live switch on a dueling net: switching Double DQN on after the fused-step and fast-path
    predict graphs exist reallocates the 1024-wide fc1 partials those graphs hold."""
    from test_gpu_double import assert_switched_on_live_equals_at_creation
    assert_switched_on_live_equals_at_creation(
        mode, lambda stream, double: make_net(6, 32, stream, double=double, mode=mode))
