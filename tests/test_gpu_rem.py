"""The random ensemble mixture head (REM) on the device against tests/rem_oracle.py, each stage fed the device's own inputs
so that errors do not carry over.  No stage uses expf or logf, so everything is bit for bit: alpha against the stated
hash at the read-back counter, theta of all three slots (slots 1 and 2 on independently computed H4), Q under alpha and
the predict Q, the targets through the row costs, the TD errors and the cost, dtheta, dZ4 and its fp16 planes, fc2's
gradient and its update under every optimizer; on both engines and both schedules, with Double DQN, prioritized replay,
n-step returns, target_steps = 0, clip_error 0 and 1 and random shift.  Also the draw counter across steps, fused runs,
graph replays and predicts, the train paths against each other, the predict paths, checkpoints, the target sync, the
refusals, the tensor-core backbone's float64 bounds and a five-step trajectory against the numpy REM step."""
import os
import random

import numpy as np
import pytest

import rem_oracle as REM
from helpers import make_args
from test_gpu_distributional import ENGINES, _L, _gather, _optimize, _ring_pair, _same_state, _slot_h4, _state

pytestmark = pytest.mark.gpu

F32 = np.float32


def _rnet(mode, A=4, K=10, clip=1.0, batch=32, hist=4, stream=None, double=False, seed=3, scale=3.0,
          optimizer="rmsprop", target_steps=10000, discount=0.99, shift=0):
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, history_length=hist, random_seed=seed, double_dqn=double, rem=True,
                                    num_heads=K, clip_error=clip, optimizer=optimizer, target_steps=target_steps,
                                    discount_rate=discount, random_shift=shift), math_mode=mode, stream=stream)
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


def _check_train_step(net, before, c0, actions, rewards, terminals, post, clip, discount=0.99, w=None, separate=True,
                      nstep=False):
    """Every stage of the last train step, bit for bit, fed the device's own inputs.  before = (weights, states) ahead
    of the step, c0 the counter it drew with; rewards / terminals are (batch, N) windows; post the poststates the
    target slots read (None: not checked, the states were shifted); separate: the target network is not the online
    one."""
    A, K, b = net.num_actions, net.num_heads, len(actions)
    assert net.mixture_counter() == c0 + 1
    al = net.last_mixture()
    assert (al == REM.alpha(net.rem_seed, c0, K)).all()
    theta = net.last_heads()
    two = net.double_dqn and separate
    h4 = net.last_activations()[3]
    w5 = before[0][4]
    assert (theta[0].reshape(b, A * K) == REM.logits(h4, w5.T)).all()
    tws = net.get_weights(which=1, with_states=False) if separate else before[0]
    if post is not None:
        assert (theta[1].reshape(b, A * K) == REM.logits(_slot_h4(net, tws, post), tws[4].T)).all()
        if two:
            assert (theta[2].reshape(b, A * K) == REM.logits(_slot_h4(net, before[0], post), w5.T)).all()
    rewards, terminals = np.asarray(rewards), np.asarray(terminals)
    returns = [REM.n_step_return(rewards[i], terminals[i], discount) for i in range(b)]
    q, _, delta, cost, g = REM.head(theta, al, actions, returns, clip, double=two, nstep=nstep, w=w)
    preq, postq = net.last_q()
    assert (preq == q[0]).all() and (postq == q[1]).all()
    if two:
        assert (net.last_online_postq() == q[2]).all()
    rc = net.last_row_costs()
    assert (rc == cost).all()
    if w is not None:
        assert (net.last_td_errors() == delta).all()
    tot = F32(0)
    for c in rc:
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(b))
    assert (net.last_head_grads() == g).all()
    dz4 = net.last_dz()[3]
    for i in range(b):
        assert (dz4[i] == REM.dz4(h4[i], w5.T, actions[i], g[i])).all(), i
    if net.math_mode == "tcgen05":
        hi16, lo16 = net.last_dz4_planes()
        ehi, elo = REM.fp16_planes(dz4)
        assert (hi16.view(np.uint16) == ehi.view(np.uint16)).all() and (lo16.view(np.uint16) == elo.view(np.uint16)).all()
    grad = REM.fc2_grad(h4, g, actions, A)
    assert (net.get_grads()[4] == grad).all()
    w_new, s_new = _optimize(net.optimizer, w5, before[1][4], grad, b)
    ws, ss = _state(net)
    assert (ws[4] == w_new).all()
    for k in range(net.num_states):
        assert (ss[4][k] == s_new[k]).all(), k
    return al, g


# ---------------------------------------------------------------------------------------------------- forward
FORWARD = [  # (mode, batch, A, K, scale)
    ("tcgen05", 1, 1, 1, 3.0), ("fp32", 64, 32, 200, 3.0), ("tcgen05", 65, 18, 10, 300.0), ("fp32", 256, 2, 2, 3.0),
]


@pytest.mark.parametrize("mode,batch,A,K,scale", FORWARD)
def test_predict_forward_stages(mode, batch, A, K, scale):
    """H4 equals a scalar twin's with the same conv and fc1 weights; theta equals the restated fp32 dot products; the
    predict Q is the mean over the heads; predict neither reads nor moves the mixture's counter; the Xavier draw is the
    scalar layout's with an (A K, 512) fc2."""
    from oracle import dqn_oracle as O
    from simple_dqn_b200 import DeepQNetwork
    fresh = DeepQNetwork(A, make_args(batch_size=batch, random_seed=5, rem=True, num_heads=K), math_mode=mode)
    for x, y in zip(fresh.get_weights(with_states=False), O.xavier_init(A * K, 5)):
        assert (x == y).all()
    net = _rnet(mode, A=A, K=K, batch=batch, scale=scale)
    twin = DeepQNetwork(A, make_args(batch_size=batch, random_seed=5), math_mode=mode)
    ws, _ = net.get_weights()
    assert ws[4].shape == (A * K, 512)
    tws = twin.get_weights(with_states=False)
    twin.set_weights(ws[:4] + [tws[4]])
    states = np.random.RandomState(batch + A).randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    q = net.predict(states)
    twin.predict(states)
    h4 = net.last_activations()[3]
    assert (h4 == twin.last_activations()[3]).all()
    theta = net.last_heads()[0]
    assert (theta.reshape(batch, A * K) == REM.logits(h4, ws[4].T)).all()
    assert (q == REM.predict_q(theta)).all()
    assert net.mixture_counter() == 0


# ---------------------------------------------------------------------------------------------------- train step
STEP = [  # (batch, A, K, n, clip, double, per, hist, discount, shift)
    (32, 4, 10, 1, 1.0, False, False, 4, 0.99, 0), (1, 1, 1, 3, 0.0, True, True, 4, 1.0, 0),
    (65, 18, 200, 1, 1.0, True, False, 4, 0.99, 0), (64, 32, 2, 3, 0.0, False, True, 4, 0.99, 0),
    (256, 2, 200, 3, 1.0, True, True, 4, 0.0, 0), (33, 4, 10, 1, 1.0, True, False, 1, 0.99, 4),
    (257, 4, 10, 1, 0.0, False, False, 4, 0.99, 0),
]


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("batch,A,K,n,clip,double,per,hist,discount,shift", STEP)
def test_train_step_stages(mode, sched, batch, A, K, n, clip, double, per, hist, discount, shift):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    from test_gpu_prioritized import _upload
    stream = Stream() if sched == "branches" else None
    ring, mem = _ring_pair(batch=batch, hist=hist, stream=stream, prioritized_replay=per, beta0=0.4, terminal_p=0.1)
    ring.actions[:] = np.random.RandomState(batch).randint(0, A, len(ring.actions))
    _upload(mem, _L().PTR_ACTIONS, ring.actions)
    mem.set_n_step(n)
    net = _rnet(mode, A=A, K=K, clip=clip, batch=batch, hist=hist, stream=stream, double=double, discount=discount,
                shift=shift)
    for step in range(2):   # the second step draws with the advanced counter
        before = _state(net)
        c0 = net.mixture_counter()
        idx = np.array(random.Random(batch * 7 + n + step).sample(range(hist, 3000 - n + 1), batch), np.int32)
        mem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, idx, n)
        al, _ = _check_train_step(net, before, c0, mb[1].astype(np.int64), mb[2], mb[4], None if shift else mb[3],
                                  clip, discount=discount, w=mem.last_weights if per else None, nstep=n > 1)
        if step == 0:
            first = al
    assert net.mixture_counter() == 2
    assert K == 1 or not (al == first).all()


@pytest.mark.parametrize("optimizer", ["rmsprop", "adam", "adadelta"])
@pytest.mark.parametrize("target_steps", [10000, 0])
def test_optimizers_and_target_steps_zero(optimizer, target_steps):
    """A host-minibatch step under every optimizer (Adam's step scalar comes from the new head), with and without a
    separate target network, Double DQN on; the engine alternates."""
    from helpers import random_minibatch
    mode = "tcgen05" if (optimizer == "adam") == (target_steps == 0) else "fp32"
    clip = 0.0 if optimizer == "adadelta" else 1.0
    net = _rnet(mode, A=4, K=10, clip=clip, batch=33, optimizer=optimizer, target_steps=target_steps, double=True)
    before = _state(net)
    pre, act, rew, post, term = random_minibatch(33, 4, 5)
    net.train((pre, act, rew, post, term))
    _check_train_step(net, before, 0, act.astype(np.int64), rew[:, None], term[:, None], post, clip,
                      separate=target_steps != 0)


# ---------------------------------------------------------------------------------------------------- the draw counter
@pytest.mark.parametrize("mode,sched", ENGINES)
def test_fused_run_equals_single_steps_and_replays_draw_fresh(mode, sched):
    """train_fused(3) equals three train_fused(1) calls (replays of the captured step graph) of a twin on an identically
    seeded ring, bit for bit; each replay draws a fresh alpha, the stated one at its counter; predict leaves the
    counter alone."""
    from simple_dqn_b200 import StateBuffer, Stream
    nets, alphas = [], []
    for single in (False, True):
        stream = Stream() if sched == "branches" else None
        _, mem = _ring_pair(stream=stream)
        net = _rnet(mode, K=10, stream=stream)
        random.seed(5)
        mem.seed_device_rng(random)
        if single:
            for step in range(3):
                net.train_fused(mem, 1)
                assert net.mixture_counter() == step + 1
                alphas.append(net.last_mixture())
                assert (alphas[-1] == REM.alpha(net.rem_seed, step, 10)).all()
        else:
            net.train_fused(mem, 3)
        nets.append(net)
    assert nets[0].mixture_counter() == 3
    assert (nets[0].last_mixture() == alphas[-1]).all()
    assert (nets[0].last_costs(3) == nets[1].last_costs(3)).all()
    _same_state(nets[0], nets[1])
    assert len({a.tobytes() for a in alphas}) == 3
    net = nets[0]
    sb = StateBuffer(make_args(), stream=net._stream_obj)
    for _ in range(4):
        sb.add(np.random.RandomState(2).randint(0, 256, (84, 84)).astype(np.uint8))
    net.predict(sb.getStateMinibatch())
    net.predict(np.random.RandomState(3).randint(0, 256, (32, 4, 84, 84)).astype(np.uint8))
    assert net.mixture_counter() == 3


# ---------------------------------------------------------------------------------------------------- paths
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_ring_step_equals_host_minibatch_step(mode):
    """Two steps from the ring (the captured step graph) equal the same steps from host tuples, bit for bit: the two
    nets draw the same alpha at the same counter."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    net = _rnet(mode, K=200, stream=stream)
    twin = _rnet(mode, K=200, stream=Stream())
    for step in range(2):
        idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
        mem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, idx, 1)
        twin.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
        assert (net.last_costs(1) == twin.last_costs(1)).all()
        assert (net.last_mixture() == twin.last_mixture()).all()
        assert (net.last_head_grads() == twin.last_head_grads()).all()
        _same_state(net, twin)
    assert net.mixture_counter() == twin.mixture_counter() == 2


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_predict_paths_agree(mode):
    """Host predict, predict_device and the captured fast path agree bit for bit on the live row; padding rows come
    back as exact zeros."""
    import ctypes as C
    from simple_dqn_b200 import StateBuffer, Stream
    stream = Stream()
    net = _rnet(mode, stream=stream)
    sb = StateBuffer(make_args(), stream=stream)
    rs = np.random.RandomState(1)
    for _ in range(4):
        sb.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    ds = sb.getStateMinibatch()
    fast = net.predict(ds)
    fast2 = net.predict(ds)
    host = net.predict(np.asarray(ds))
    L = _L()
    qp = net.device_view(L.NET_PTR_Q_ONLINE, (32, 4)).ptr
    L.call("b200dqn_net_predict_device", net._h, C.c_void_p(ds.device_ptr()), 1, C.c_void_p(qp), net._stream)
    dev = net._read_f32(L.NET_PTR_Q_ONLINE, (32, 4))
    assert (fast[0] == host[0]).all() and (fast2 == fast).all() and (dev[0] == host[0]).all()
    assert (fast[1:] == 0).all() and (dev[1:] == 0).all()
    assert (host[0] != 0).any()
    assert net.mixture_counter() == 0


# ---------------------------------------------------------------------------------------------------- state
def test_checkpoints_target_sync_and_refusals(tmp_path):
    """Both checkpoint layouts round-trip; a scalar checkpoint does not load, nor the reverse; a QR checkpoint with as
    many quantiles as heads has the same fc2 shape and loads; the target sync copies fc2's weights and states; the
    refusals; and a REM step launches one kernel more than a QR step (the mixture draw)."""
    from helpers import random_minibatch
    from simple_dqn_b200 import DeepQNetwork, Stream
    from test_gpu_quantile import _qnet
    net = _rnet("tcgen05", optimizer="adam")
    net.train(random_minibatch(32, 4, 3))
    for layout in ("neon-1.3.0", "pre-1.0"):
        path = os.path.join(str(tmp_path), "rem_%s.pkl" % layout)
        net.save_weights(path, layout=layout)
        other = _rnet("fp32", optimizer="adam", seed=9)
        other.load_weights(path)
        _same_state(net, other)
        scalar = DeepQNetwork(4, make_args(), math_mode="tcgen05")
        with pytest.raises(AssertionError):
            scalar.load_weights(path)
        spath = os.path.join(str(tmp_path), "scalar.pkl")
        scalar.save_weights(spath, layout=layout)
        with pytest.raises(AssertionError):
            other.load_weights(spath)
    qr = _qnet("tcgen05", nq=10, optimizer="adam")
    qpath = os.path.join(str(tmp_path), "qr.pkl")
    qr.save_weights(qpath)
    net.load_weights(qpath)
    assert (net.get_weights(with_states=False)[4] == qr.get_weights(with_states=False)[4]).all()
    net.update_target_network()
    assert (net.get_weights(which=1, with_states=False)[4] == net.get_weights(with_states=False)[4]).all()
    L = _L()
    for k in range(net.num_states):
        a, b = np.empty((4 * 10, 512), F32), np.empty((4 * 10, 512), F32)
        L.call("b200dqn_net_get_state", net._h, 0, 4, k, L.np_ptr(a), None)
        L.call("b200dqn_net_get_state", net._h, 1, 4, k, L.np_ptr(b), None)
        assert (a == b).all()
    for kw in ({"num_heads": 0}, {"num_heads": 201}, {"quantile_regression": True, "num_quantiles": 10},
               {"distributional": True, "num_atoms": 51}, {"implicit_quantiles": True, "num_tau_samples": 8}):
        args = dict(rem=True, num_heads=10)
        args.update(kw)
        with pytest.raises(AssertionError):
            DeepQNetwork(4, make_args(**args), math_mode="tcgen05")
    for kw in ({"dueling": True}, {"munchausen": True}):
        with pytest.raises(NotImplementedError, match="REM"):
            DeepQNetwork(4, make_args(rem=True, num_heads=10, **kw), math_mode="tcgen05")
    with pytest.raises(NotImplementedError, match="REM"):
        net.comm_init(bytes(128), 0, 2)
    with pytest.raises(AssertionError):
        net.last_deltas()
    for sel in (L.NET_PTR_QUANTILES, L.NET_PTR_LOGITS, L.NET_PTR_IQN_TAU_COUNTER):
        with pytest.raises(AssertionError):
            net._read_f32(sel, (1,))
    with pytest.raises(AssertionError):
        qr.last_mixture()
    for mode in ("tcgen05", "fp32"):
        stream = Stream()
        _, mem = _ring_pair(stream=stream)
        random.seed(1)
        mem.seed_device_rng(random)
        counts = []
        for head in ("qr", "rem"):
            n = _qnet(mode, stream=stream) if head == "qr" else _rnet(mode, stream=stream)
            n.train_fused(mem, 1)
            counts.append(n.launches_per_step())
        assert counts[1] == counts[0] + 1, counts


# ---------------------------------------------------------------------------------------------------- rest of the net
@pytest.mark.parametrize("batch,sched", [(1, "serial"), (65, "branches")])
def test_backbone_kernels_within_float64_bounds(batch, sched):
    """With dZ4 from the REM head, every tensor-core kernel of the step stays inside the float64 bound its hi/lo scheme
    promises (tests/test_gpu_kernels.py's yardstick), forward and backward."""
    import kernel_ref as K
    from helpers import random_minibatch
    from simple_dqn_b200 import Stream
    from test_gpu_kernels import _chain, _check
    net = _rnet("tcgen05", K=200, batch=batch, stream=Stream() if sched == "branches" else None, double=True)
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


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_fused_trajectory_against_a_numpy_rem_step(mode):
    """Five fused steps against tests/rem_oracle.numpy_step (oracle.dqn_oracle's forward, backward and RMSProp with the
    REM head) on the same minibatches and the same stated alpha: cost within 1e-3, every layer's update within rel-L2
    2e-2.  At the default K = 200: with K = 10 this seed's trajectory is ill-conditioned (a 1e-6 relative perturbation
    of the initial weights moves the numpy step's fifth conv1 update by 3.5e-2), so no engine could be held to it."""
    from helpers import rel_l2
    from simple_dqn_b200 import Stream
    from test_gpu_prioritized import _dev
    stream = Stream()
    ring, mem = _ring_pair(stream=stream, terminal_p=0.05)
    net = _rnet(mode, K=200, stream=stream)
    ws, ss = _state(net)
    ows, oss = [w.copy() for w in ws], [s[0].copy() for s in ss]
    tws = net.get_weights(which=1, with_states=False)
    w0 = [w.copy() for w in ws]
    random.seed(9)
    mem.seed_device_rng(random)
    for step in range(5):
        net.train_fused(mem, 1)
        idx = _dev(mem, _L().PTR_INDEXES, np.int32, 32).astype(np.int64)
        mb = _gather(ring, idx, 1)
        al = REM.alpha(net.rem_seed, step, 200)
        assert (net.last_mixture() == al).all()
        ref, _, _ = REM.numpy_step(ows, oss, tws, (mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]), 200, al)
        cost = float(net.last_costs(1)[0])
        assert abs(cost - ref) <= 1e-3 * abs(ref), (cost, ref)
    got = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(got[l] - w0[l], ows[l] - w0[l]) <= 2e-2, l
