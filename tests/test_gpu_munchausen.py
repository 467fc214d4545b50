"""The Munchausen DQN target on the device against tests/munchausen_oracle.py, each stage fed the device's own inputs so
that errors do not carry over: the target network's Q on the prestates (the extra one-slot pass) bit for bit against a
twin's predict, the target y within one fp32 ulp of the restated rules on the device's own Q rows (the device's fp64 exp
and log are not the C library's), and everything downstream of y bit for bit (delta, row costs, TD errors, cost, dZ4 and
its fp16 planes, fc2's gradient and its update under every optimizer), on both engines and both schedules, with
prioritized replay, n-step returns and target_steps = 0.  Also: one action against the scalar head over five fused
steps, the launch counts, a five-step trajectory against the numpy step, the train paths against each other, the target
sync under captured step graphs, predict, checkpoints, the refusals and the backbone's float64 bounds."""
import os
import random

import numpy as np
import pytest

import head_oracle as H
import munchausen_oracle as M
from helpers import make_args
from test_gpu_distributional import ENGINES, _L, _gather, _optimize, _ring_pair, _same_state, _state

pytestmark = pytest.mark.gpu

F32 = np.float32
MARGS = dict(munchausen_alpha=0.9, munchausen_tau=0.03, munchausen_clip=-1.0)


def _mnet(mode, A=4, batch=32, hist=4, stream=None, seed=3, scale=3.0, optimizer="rmsprop", target_steps=10000,
          discount=0.99, munchausen=True, **kw):
    """A net whose weights make Q spreads of a few units (the soft-max is neither one-hot nor flat at tau = 0.03), with
    non-zero optimizer states and a target network that differs from the online one.  munchausen=False: the scalar net
    with the same weights."""
    from simple_dqn_b200 import DeepQNetwork
    m = dict(MARGS, **kw)
    net = DeepQNetwork(A, make_args(batch_size=batch, history_length=hist, random_seed=seed, optimizer=optimizer,
                                    target_steps=target_steps, discount_rate=discount, munchausen=munchausen, **m),
                       math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(scale)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [[np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for _ in range(net.num_states)]
                         for w in ws])
    if target_steps:
        net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                        None, which=1)
    return net


def _predict_with(net, weights, states):
    """Q of `weights` on `states` from a scalar twin's predict: the independent source for every Q row of the step."""
    from simple_dqn_b200 import DeepQNetwork
    twin = DeepQNetwork(net.num_actions, make_args(batch_size=net.batch_size, history_length=net.history_length),
                        math_mode=net.math_mode)
    twin.set_weights(list(weights))
    return twin.predict(states)


EXACT = []   # per checked step: the fraction of targets equal to the restatement's


def _check_train_step(net, before, pre, post, actions, returns, nstep, w=None, td=False, separate=True, margs=MARGS):
    """Every stage of the last train step.  before = (weights, states) ahead of the step, returns the per-sample (R, g)
    (g = 0 at a terminal), nstep: the n-step form of the target's last operation."""
    A, b = net.num_actions, len(actions)
    actions = np.asarray(actions, np.int64)
    tws = net.get_weights(which=1, with_states=False) if separate else before[0]
    preq, postq = net.last_q()
    qpre = net.last_target_q_pre()
    # the Q rows: slot 0 online on the prestates, slot 1 target on the poststates, slot 2 (the pass) target on the
    # prestates, each bit for bit against a twin's predict
    assert (preq == _predict_with(net, before[0], pre)).all()
    assert (postq == _predict_with(net, tws, post)).all()
    if separate:
        assert (qpre == _predict_with(net, tws, pre)).all()
    else:
        assert (qpre == preq).all()
    # y within one fp32 ulp of the rules on the device's rows
    y = net.last_td_targets()
    ref = M.targets(postq, qpre, actions, returns, margs["munchausen_alpha"], margs["munchausen_tau"],
                    margs["munchausen_clip"], nstep)
    assert (np.abs(y.astype(np.float64) - ref) <= np.spacing(np.abs(ref))).all(), np.abs(y - ref).max()
    EXACT.append(float((y == ref).mean()))
    # downstream of the device's own y: the scalar head, bit for bit
    d = (preq[np.arange(b), actions] - y).astype(F32)
    if w is None:
        rc = (F32(0.5) * d * d).astype(F32)
    else:
        wb = np.asarray(w, F32)
        rc = (wb * (F32(0.5) * d * d)).astype(F32)
    if td:
        assert (net.last_td_errors() == d).all()
    assert (net.last_row_costs() == rc).all()
    tot = F32(0)
    for c in rc:
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(b))
    clip = F32(net.clip_error or 0)
    dc = np.minimum(np.maximum(d, -clip), clip).astype(F32) if clip > 0 else d
    if w is not None:
        dc = (dc * wb).astype(F32)
    deltas = np.zeros((b, A), F32)
    deltas[np.arange(b), actions] = dc
    assert (net.last_deltas() == deltas).all()
    h4 = net.last_activations()[3]
    w5 = before[0][4]
    dz4 = np.where(h4 > 0, (dc[:, None] * w5[actions]).astype(F32), F32(0)).astype(F32)
    got = net.last_dz()[3]
    assert (got == dz4).all()
    if net.math_mode == "tcgen05":
        import c51_oracle as C51
        hi16, lo16 = net.last_dz4_planes()
        ehi, elo = C51.fp16_planes(dz4)
        assert (hi16.view(np.uint16) == ehi.view(np.uint16)).all() and (lo16.view(np.uint16) == elo.view(np.uint16)).all()
    grad = H.fc2_grad(h4, dc, actions, A)
    assert (net.get_grads()[4] == grad).all()
    w_new, s_new = _optimize(net.optimizer, w5, before[1][4], grad, b)
    ws, ss = _state(net)
    assert (ws[4] == w_new).all()
    for k in range(net.num_states):
        assert (ss[4][k] == s_new[k]).all(), k
    return y


# ---------------------------------------------------------------------------------------------------- train step
STEP = [  # (batch, A, n, per, hist, alpha, tau, l0)
    (32, 4, 1, False, 4, 0.9, 0.03, -1.0), (1, 1, 3, True, 4, 0.9, 0.03, -1.0), (64, 18, 1, False, 4, 1.0, 1.0, 0.0),
    (65, 32, 3, True, 4, 0.9, 0.03, -1.0), (257, 2, 1, False, 4, 0.0, 1e-3, -1.0), (33, 18, 3, False, 1, 0.9, 0.03, -0.5),
]


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("batch,A,n,per,hist,alpha,tau,l0", STEP)
def test_train_step_stages(mode, sched, batch, A, n, per, hist, alpha, tau, l0):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    from test_gpu_prioritized import _upload
    stream = Stream() if sched == "branches" else None
    ring, mem = _ring_pair(batch=batch, hist=hist, stream=stream, prioritized_replay=per, beta0=0.4, terminal_p=0.1)
    ring.actions[:] = np.random.RandomState(batch).randint(0, A, len(ring.actions))
    _upload(mem, _L().PTR_ACTIONS, ring.actions)
    mem.set_n_step(n)
    margs = dict(munchausen_alpha=alpha, munchausen_tau=tau, munchausen_clip=l0)
    net = _mnet(mode, A=A, batch=batch, hist=hist, stream=stream, **margs)
    before = _state(net)
    idx = np.array(random.Random(batch * 7 + n).sample(range(hist, 3000 - n + 1), batch), np.int32)
    mem.set_indexes(idx)
    net.train(DeviceMinibatch(mem, sampled=True))
    mb = _gather(ring, idx, n)
    import c51_oracle as C51
    returns = [C51.n_step_return(mb[2][i], mb[4][i], 0.99) for i in range(batch)]
    _check_train_step(net, before, mb[0], mb[3], mb[1], returns, n > 1, w=mem.last_weights if per else None, td=per,
                      margs=margs)


@pytest.mark.parametrize("optimizer", ["rmsprop", "adam", "adadelta"])
@pytest.mark.parametrize("target_steps", [10000, 0])
def test_optimizers_and_target_steps_zero(optimizer, target_steps):
    """A host-minibatch step under every optimizer (Adam's step scalar comes from the new head), with and without a
    separate target network (without one, slot 0's row is the prestate policy and no pass runs); the engine
    alternates."""
    from helpers import random_minibatch
    import c51_oracle as C51
    mode = "tcgen05" if (optimizer == "adam") == (target_steps == 0) else "fp32"
    net = _mnet(mode, A=4, batch=33, optimizer=optimizer, target_steps=target_steps)
    before = _state(net)
    pre, act, rew, post, term = random_minibatch(33, 4, 5)
    net.train((pre, act, rew, post, term))
    returns = [C51.one_step_return(rew[i], term[i], 0.99) for i in range(33)]
    _check_train_step(net, before, pre, post, act, returns, False, separate=target_steps != 0)


# ---------------------------------------------------------------------------------------------------- identities
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
@pytest.mark.parametrize("n", [1, 3])
def test_one_action_equals_the_scalar_head(mode, n):
    """A = 1: pi = 1 and tau ln pi = 0 exactly, so five fused Munchausen steps equal five scalar steps bit for bit in
    weights, optimizer states and costs, although the Munchausen step runs the extra pass."""
    from simple_dqn_b200 import Stream
    from test_gpu_prioritized import _upload
    nets = []
    for munchausen in (True, False):
        stream = Stream()
        ring, mem = _ring_pair(stream=stream)
        ring.actions[:] = 0
        _upload(mem, _L().PTR_ACTIONS, ring.actions)
        mem.set_n_step(n)
        net = _mnet(mode, A=1, stream=stream, munchausen=munchausen)
        random.seed(5)
        mem.seed_device_rng(random)
        net.train_fused(mem, 5)
        nets.append(net)
    assert (nets[0].last_costs(5) == nets[1].last_costs(5)).all()
    _same_state(nets[0], nets[1])


def test_launch_counts_and_refusals():
    """The pass adds conv1_fwd, conv23_fwd (or conv2_fwd and conv3_fwd above 64 rows) and fc1_fwd on the tensor-core
    engine, the four forward GEMMs on the SIMT one; with target_steps = 0 nothing is added.  set_double_q and comm_init
    refuse a Munchausen net, and the Munchausen selectors refuse any other net."""
    from simple_dqn_b200 import DeepQNetwork, Stream
    for mode in ("tcgen05", "fp32"):
        for batch in (32, 65):
            stream = Stream()
            _, mem = _ring_pair(batch=batch, stream=stream)
            random.seed(1)
            mem.seed_device_rng(random)
            counts = []
            for kw in (dict(munchausen=False), dict(), dict(target_steps=0)):
                net = _mnet(mode, batch=batch, stream=stream, **kw)
                net.train_fused(mem, 1)
                counts.append(net.launches_per_step())
            extra = 4 if mode == "fp32" or batch > 64 else 3
            assert counts == [counts[0], counts[0] + extra, counts[0]], (mode, batch, counts)
    net = _mnet("tcgen05")
    with pytest.raises(AssertionError, match="Munchausen"):
        net.set_double_dqn(True)
    with pytest.raises(AssertionError, match="Munchausen"):
        DeepQNetwork(4, make_args(munchausen=True, double_dqn=True), math_mode="fp32")
    with pytest.raises(NotImplementedError, match="Munchausen"):
        net.comm_init(bytes(128), 0, 2)
    scalar = DeepQNetwork(4, make_args(), math_mode="fp32")
    for f in (scalar.last_td_targets, scalar.last_target_q_pre):
        with pytest.raises(AssertionError, match="Munchausen"):
            f()


# ---------------------------------------------------------------------------------------------------- paths
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_train_paths_agree_and_target_sync(mode):
    """Ring steps (the captured step graph) equal host-minibatch steps; train_fused equals sample + train_sampled and
    step_host; after a target sync inside the cached graphs the pass's row equals the online one, bit for bit."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    net = _mnet(mode, stream=stream)
    twin = _mnet(mode, stream=Stream())
    for step in range(2):
        idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
        mem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, idx, 1)
        twin.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
        assert (net.last_costs(1) == twin.last_costs(1)).all()
        assert (net.last_td_targets() == twin.last_td_targets()).all()
        _same_state(net, twin)
    streams = [Stream() for _ in range(3)]
    mems = [_ring_pair(stream=s)[1] for s in streams]
    nets = [_mnet(mode, stream=s) for s in streams]
    random.seed(4)
    mems[0].seed_device_rng(random)
    key = mems[0].read_device_rng()
    for m in mems[1:]:
        _L().call("b200dqn_replay_set_rng", m._h, _L().np_ptr(key), m._stream)
        m._rng_on_device = True
    empty = np.zeros((0, 84, 84), np.uint8)
    for step in range(4):
        if step == 2:
            for x in nets:
                x.update_target_network()
        nets[0].train_fused(mems[0], 1)
        mems[1].sample()
        nets[1].train(DeviceMinibatch(mems[1], sampled=True))
        nets[2].step_host(mems[2], [], [], empty, [], train_repeat=1)
        for x in nets[1:]:
            assert (x.last_costs(1) == nets[0].last_costs(1)).all()
            _same_state(x, nets[0])
        if step == 2:   # the step right after the sync: target and online weights are equal
            assert (nets[0].last_target_q_pre() == nets[0].last_q()[0]).all()
        elif step < 2:
            assert (nets[0].last_target_q_pre() != nets[0].last_q()[0]).any()


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_predict_and_checkpoints_match_the_scalar_net(mode, tmp_path):
    """Predict is the scalar head's (same weights, same Q bits); checkpoints load both ways between Munchausen and scalar
    nets."""
    net = _mnet(mode)
    scalar = _mnet(mode, munchausen=False, seed=8)
    scalar.set_weights(net.get_weights(with_states=False))
    states = np.random.RandomState(2).randint(0, 256, (32, 4, 84, 84)).astype(np.uint8)
    assert (net.predict(states) == scalar.predict(states)).all()
    from helpers import random_minibatch
    net.train(random_minibatch(32, 4, 3))
    for src, dst in ((net, _mnet(mode, munchausen=False, seed=9)), (scalar, _mnet(mode, seed=9))):
        path = os.path.join(str(tmp_path), "ckpt.pkl")
        src.save_weights(path)
        dst.load_weights(path)
        _same_state(src, dst)


# ---------------------------------------------------------------------------------------------------- rest of the net
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_fused_trajectory_against_a_numpy_munchausen_step(mode):
    """Five fused steps against tests/munchausen_oracle.numpy_step on the same minibatches: cost within 1e-3, every
    layer's update within rel-L2 3e-2.  The bar is wider than the scalar head's 2e-2: y moves with the Q rows by up to
    alpha + gamma (the bonus adds alpha times the log-policy's derivative, itself bounded by 1) where the scalar target
    moves by gamma, so about twice the engine's rounding reaches the deltas."""
    from helpers import rel_l2
    from simple_dqn_b200 import Stream
    from test_gpu_prioritized import _dev
    stream = Stream()
    ring, mem = _ring_pair(stream=stream, terminal_p=0.05)
    net = _mnet(mode, stream=stream)
    ws, ss = _state(net)
    ows, oss = [w.copy() for w in ws], [s[0].copy() for s in ss]
    tws = net.get_weights(which=1, with_states=False)
    w0 = [w.copy() for w in ws]
    random.seed(9)
    mem.seed_device_rng(random)
    for _ in range(5):
        net.train_fused(mem, 1)
        idx = _dev(mem, _L().PTR_INDEXES, np.int32, 32).astype(np.int64)
        mb = _gather(ring, idx, 1)
        ref, _, _ = M.numpy_step(ows, oss, tws, (mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
        cost = float(net.last_costs(1)[0])
        assert abs(cost - ref) <= 1e-3 * abs(ref), (cost, ref)
    got = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(got[l] - w0[l], ows[l] - w0[l]) <= 3e-2, l


@pytest.mark.parametrize("batch,sched", [(1, "serial"), (65, "branches")])
def test_backbone_kernels_within_float64_bounds(batch, sched):
    """With dZ4 from the Munchausen head, every tensor-core kernel of the step stays inside the float64 bound its hi/lo
    scheme promises (tests/test_gpu_kernels.py's yardstick), forward and backward.  The pass's Q row equals a twin's
    predict bit for bit (test_train_step_stages), so its kernels are held to the same bounds through the twin."""
    import kernel_ref as K
    from helpers import random_minibatch
    from simple_dqn_b200 import Stream
    from test_gpu_kernels import _chain, _check
    net = _mnet("tcgen05", batch=batch, stream=Stream() if sched == "branches" else None)
    net.keep_grads(True)
    ws = net.get_weights(with_states=False)
    mb = random_minibatch(batch, 4, 7)
    net.train(mb)
    pre = mb[0]
    h1, h2, h3, h4 = net.last_activations()
    dz1, dz2, dz3, dz4 = net.last_dz()
    assert np.abs(dz4).max() > 0
    grads = net.get_grads()
    c = lambda k: _chain("tcgen05", k, batch, 4)
    fc1_dgrad = lambda a, b: K.fc_dgrad(a, b).reshape(len(a), 64, 7, 7)
    r = {}
    r.update(_check("conv1_fwd", "tcgen05", K.conv_fwd(0), K.states_f64(pre), ws[0], h1, c("conv1_fwd"), post=K.relu,
                    a_exact=True))
    r.update(_check("conv2_fwd", "tcgen05", K.conv_fwd(1), h1, ws[1], h2, c("conv2_fwd"), post=K.relu))
    r.update(_check("conv3_fwd", "tcgen05", K.conv_fwd(2), h2, ws[2], h3, c("conv3_fwd"), post=K.relu))
    r.update(_check("fc1_fwd", "tcgen05", K.fc_fwd, h3, ws[3], h4, c("fc1_fwd"), post=K.relu))
    r.update(_check("fc1_dgrad", "tcgen05", fc1_dgrad, dz4, ws[3], dz3, c("fc1_dgrad"), mask=h3 > 0))
    r.update(_check("conv3_dgrad", "tcgen05", K.conv_dgrad(2), dz3, ws[2], dz2, c("conv3_dgrad"), mask=h2 > 0))
    r.update(_check("conv2_dgrad", "tcgen05", K.conv_dgrad(1), dz2, ws[1], dz1, c("conv2_dgrad"), mask=h1 > 0))
    r.update(_check("fc1_wgrad", "tcgen05", K.fc_wgrad, h3, dz4, grads[3], c("fc1_wgrad")))
    r.update(_check("conv3_wgrad", "tcgen05", K.conv_wgrad(2), h2, dz3, grads[2], c("conv3_wgrad")))
    r.update(_check("conv2_wgrad", "tcgen05", K.conv_wgrad(1), h1, dz2, grads[1], c("conv2_wgrad")))
    r.update(_check("conv1_wgrad", "tcgen05", K.conv_wgrad(0), K.states_f64(pre), dz1, grads[0], c("conv1_wgrad"),
                    a_exact=True))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, bad


def test_report_exact_fraction():
    """The share of device targets equal to the restatement's bit for bit, over every checked step (printed; the
    assertion is the one-ulp bound in _check_train_step)."""
    if EXACT:
        print("munchausen targets equal to the restatement: %.4f over %d steps" % (float(np.mean(EXACT)), len(EXACT)))
