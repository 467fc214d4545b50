"""The implicit quantile network head (IQN) on the device against tests/iqn_oracle.py, each stage fed the device's own
inputs so that errors do not carry over: tau from the stated hash at the device's counter, the cosine features within
one fp32 ulp, and bit for bit phi, X, theta, Q, T, the row costs, the TD errors, the cost, dtheta, dZ4 and its fp16
planes, fc2's gradient, dpsi, dphi, dWe and the embedding's update; fc1's forward, dgrad and wgrad at the expanded rows
and conv3's wgrad from dpsi within the float64 bounds of tests/kernel_ref.py.  Both engines and both schedules, with
Adam, Adadelta, target_steps = 0, kappa 0, first-index ties of a*, importance weights with n-step returns and up to 4096
expanded rows; every train path against the others, the predict paths, checkpoints, the target sync, the refusals,
launch counts and a five-step trajectory against the numpy IQN step."""
import numpy as np
import pytest

import c51_oracle as C51
import iqn_oracle as IQ
import kernel_ref as K
from helpers import make_args, random_minibatch, rel_l2
from test_gpu_distributional import _gather, _optimize, _ring_pair
from test_gpu_kernels import _chain, _check

pytestmark = pytest.mark.gpu

F32 = np.float32
# fc1's input column n in Neon's (c, p, q) order sits at internal column (p * 7 + q) * 64 + c
PERM = np.array([((n // 7 % 7) * 7 + n % 7) * 64 + n // 49 for n in range(3136)])


def _inet(A=4, N=8, K=32, batch=8, kappa=1.0, stream=None, optimizer="rmsprop", target_steps=10000, seed=3,
          mode="fp32", tie=False):
    """tie: the target network's fc2 rows are all equal, so every target Q of a sample ties and a* must be action 0."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, random_seed=seed, implicit_quantiles=True, num_tau_samples=N,
                                    num_quantile_samples=K, clip_error=kappa, optimizer=optimizer,
                                    target_steps=target_steps), math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [[np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for _ in range(net.num_states)]
                         for w in ws])
    if target_steps:
        tws = [(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws]
        if tie:
            tws[4][:] = tws[4][:1]
        net.set_weights(tws, None, which=1)
    return net


def _read(net, which, shape, dtype=F32):
    from simple_dqn_b200 import _lib as L
    return L.download(net.device, net.device_view(which, shape).ptr, shape, dtype, net._stream)


def _counter(net):
    from simple_dqn_b200 import _lib as L
    return int(_read(net, L.NET_PTR_IQN_TAU_COUNTER, (1,), np.uint64)[0])


def _check_step(net, before, tws, actions, returns, c0, kappa, w=None, t=1):
    """Every stage of the last train step.  before: (weights, states) of the online net ahead of the step; tws the
    target weights; returns per-sample (R, g); c0 the counter the step drew with."""
    from simple_dqn_b200 import _lib as L
    A, N, B = net.num_actions, net.num_tau_samples, net.batch_size
    R, ld = B * N, net._iqn_rows()
    ws, ss = before
    assert _counter(net) == c0 + 1
    tau = net.last_taus()
    assert (tau[:, :R] == IQ.tau_draw(net.tau_seed, c0, 2, B, N)).all()
    assert (tau[:, :R] > 0).all() and (tau[:, :R] < 1).all()
    c = _read(net, L.NET_PTR_IQN_COS, (2, ld, 64))[:, :R]
    ref = np.cos((np.pi * np.arange(64)) * tau[:, :R, None].astype(np.float64))
    assert (np.abs(c - ref) <= np.spacing(np.abs(ref).astype(F32))).all()
    phi = _read(net, L.NET_PTR_IQN_PHI, (2, ld, 3136))[:, :R]
    for z, wz in ((0, ws), (1, tws)):
        assert (phi[z] == IQ.phi(c[z], _we_internal(wz[5]))).all(), z
    x = _read(net, L.NET_PTR_IQN_X, (2, ld, 3136))[:, :R]
    h3 = _read(net, L.NET_PTR_H3, (B, 3136))
    assert (x[0] == IQ.modulate(h3, phi[0], N)).all()
    # fc1 on X within the float64 bound of its engine's scheme, at the expanded row count
    mode = net.math_mode
    h4 = _read(net, L.NET_PTR_H4, (ld, 512))[:R]
    xn = x[0][:, PERM]                     # fc1's input in Neon's (c, p, q) column order
    ratios = _check("fc1_fwd", mode, K.fc_fwd, xn, ws[3], h4, _chain(mode, "fc1_fwd", R, 4), post=K.relu)
    theta = net.last_iqn_quantiles()[:, :R]
    assert (theta[0] == IQ.logits(h4, ws[4].T)).all()
    q0, q1, astar, T, loss, g = IQ.head(theta, tau[0], actions, returns, kappa, N, w)
    preq, postq = net.last_q()
    assert (preq == q0).all() and (postq == q1).all()
    assert (net.last_iqn_target_quantiles() == T).all()
    assert (net.last_iqn_quantile_grads() == g).all()
    rc = net.last_row_costs()
    assert (rc == (loss if w is None else (np.asarray(w, F32) * loss).astype(F32))).all()
    cost = F32(0)
    for v in rc:
        cost = F32(cost + v)
    assert net.last_costs(1)[0] == cost / F32(B)
    if w is not None:   # a prioritized ring: the priority update gets the unweighted row loss
        assert (net.last_td_errors() == loss).all()
    dz4 = _read(net, L.NET_PTR_DZ4, (ld, 512))[:R]
    assert (dz4 == IQ.dz4(h4, ws[4].T, actions, g, N)).all()
    if mode == "tcgen05":   # the planes the tensor-core fc1 dgrad and wgrad read
        p = net.device_view(L.NET_PTR_DZ4_PLANES, (1,)).ptr
        lo_off = _plane_lo_off(net)
        hi16 = L.download(net.device, p, (R, 512), np.float16, net._stream)
        lo16 = L.download(net.device, p + 2 * lo_off, (R, 512), np.float16, net._stream)
        ehi, elo = C51.fp16_planes(dz4)
        assert (hi16.view(np.uint16) == ehi.view(np.uint16)).all() and (lo16.view(np.uint16) == elo.view(np.uint16)).all()
    grads = net.get_grads()
    assert (grads[4] == IQ.fc2_grad(h4, actions, g, N, A)).all()
    dx = _read(net, L.NET_PTR_IQN_DX, (ld, 3136))[:R]
    ratios.update(_check("fc1_dgrad", mode, K.fc_dgrad, dz4, ws[3], dx[:, PERM], _chain(mode, "fc1_dgrad", R, 4),
                         mask=xn > 0))
    # the tensor-core engine reduces fc1's wgrad in chunks of 256 expanded rows, one partial each, summed in fp32
    nw = _chain(mode, "fc1_wgrad", min(R, 256), 4) + -(-R // 256) if mode == "tcgen05" else R
    ratios.update(_check("fc1_wgrad", mode, K.fc_wgrad, xn, dz4, grads[3], nw))
    dpsi, dphi = IQ.mod_bwd(dx, phi[0], h3, N)
    assert (_read(net, L.NET_PTR_DZ3, (B, 3136)) == dpsi).all()
    h2 = net.last_activations()[1]
    ratios.update(_check("conv3_wgrad", mode, K.conv_wgrad(2), h2, dpsi.reshape(B, 7, 7, 64).transpose(0, 3, 1, 2),
                         grads[2], _chain(mode, "conv3_wgrad", B, 4)))
    assert max(ratios.values()) <= 1.0, ratios
    assert (_read(net, L.NET_PTR_IQN_DPHI, (ld, 3136))[:R] == dphi).all()
    dwe = IQ.we_grad(c[0], dphi)
    assert (grads[5] == dwe[:, PERM].T).all()
    w1, s1 = net.get_weights()[0], net.get_states()
    for layer, gl in ((4, grads[4]), (5, grads[5])):
        ew, es = _optimize(net.optimizer, ws[layer], ss[layer], gl, B, t)
        assert (w1[layer] == ew).all(), layer
        for p, q in zip(s1[layer], es):
            assert (p == q).all(), layer
    return astar, loss


def _plane_lo_off(net):
    """Offset (elements) of dZ4's lo plane: the planes are reserved for every expanded row."""
    import ctypes as C
    from simple_dqn_b200 import _lib as L
    p, b = C.c_void_p(), C.c_size_t()
    L.call("b200dqn_net_device_ptr", net._h, L.NET_PTR_DZ4_PLANES, C.byref(p), C.byref(b))
    return b.value // 2 - net.batch_size * 512


def _we_internal(we_neon):
    """(3136, 64) Neon embedding -> (64, 3136) in fc1's internal column order."""
    out = np.empty((64, 3136), F32)
    out[:, PERM] = we_neon.T
    return out


def _states(net):
    return [[a.copy() for a in s] for s in net.get_states()]


ENGINES = ["tcgen05", "fp32"]
STEP = [  # (batch, A, N, K, kappa, optimizer, target_steps, tie): 8-512 expanded rows cross fc1's split counts,
    # 32 / 64 samples conv23 and 65 the two-kernel conv2 / conv3 path of the tensor-core engine
    (8, 4, 8, 32, 1.0, "rmsprop", 10000, False), (1, 1, 1, 1, 1.0, "rmsprop", 10000, False),
    (5, 2, 64, 1, 0.0, "adam", 10000, True), (32, 18, 8, 32, 1.0, "adadelta", 0, False),
    (64, 32, 64, 32, 1.0, "rmsprop", 10000, False), (3, 4, 8, 8, 0.5, "adam", 0, False),
    (65, 4, 8, 1, 1.0, "rmsprop", 10000, True),
]


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
@pytest.mark.parametrize("batch,A,N,K,kappa,optimizer,ts,tie", STEP)
def test_train_step_stages(mode, sched, batch, A, N, K, kappa, optimizer, ts, tie):
    from simple_dqn_b200 import Stream
    stream = Stream() if sched == "branches" else None
    net = _inet(A, N, K, batch, kappa, stream, optimizer, ts, mode=mode, tie=tie)
    assert len(net.layer_shapes()) == 6 and net.layer_shapes()[5] == (3136, 64)
    for step in range(2):
        pre, act, rew, post, term = random_minibatch(batch, A, seed=10 + step)
        before = (net.get_weights()[0], _states(net))
        tws = net.get_weights(which=1, with_states=False) if ts else before[0]
        c0 = _counter(net)
        net.train((pre, act, rew, post, term))
        returns = [IQ.one_step_return(rew[i], term[i], 0.99) for i in range(batch)]
        astar, _ = _check_step(net, before, tws, act, returns, c0, kappa, t=step + 1)
        if tie:
            assert (astar == 0).all()


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
def test_weighted_nstep_step_stages(mode, sched):
    """A step on a prioritized ring with n-step 3: the importance-weighted dtheta and row costs and the unweighted TD
    errors, with every other stage, bit for bit."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    import random
    stream = Stream() if sched == "branches" else None
    B, A, N = 16, 4, 8
    ring, mem = _ring_pair(batch=B, stream=stream, prioritized_replay=True, beta0=0.4, terminal_p=0.1)
    mem.set_n_step(3)
    net = _inet(A, N, 32, B, 1.0, stream, mode=mode)
    idx0 = np.array(random.Random(0).sample(range(4, 2990), B), np.int32)
    for step in range(2):
        idx = np.roll(idx0, step)   # the second step draws slots the first gave their own priorities
        mem.set_indexes(idx)
        before = (net.get_weights()[0], _states(net))
        tws = net.get_weights(which=1, with_states=False)
        c0 = _counter(net)
        net.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, idx, 3)
        w = mem.last_weights
        returns = [IQ.n_step_return(mb[2][i], mb[4][i], 0.99) for i in range(B)]
        _check_step(net, before, tws, mb[1].astype(np.int64), returns, c0, 1.0, w=w, t=step + 1)
        if step:
            assert (w != F32(1)).any()


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
def test_fused_equals_sampled_path(mode, sched):
    """Prioritized replay with n-step 3: two steps inside one train_fused(2) draw the generator's next two taus, and
    equal two sample-then-train_sampled steps bit for bit."""
    import random
    from simple_dqn_b200 import Stream
    stream = Stream() if sched == "branches" else None
    B, A, N = 8, 4, 8
    nets, mems = [], []
    for _ in range(2):
        mem = _ring_pair(batch=B, stream=stream, prioritized_replay=True, beta0=0.4, terminal_p=0.1)[1]
        mem.set_n_step(3)
        mems.append(mem)
        nets.append(_inet(A, N, 32, B, 1.0, stream, mode=mode))
    random.seed(5)
    mems[0].seed_device_rng(random)
    c0 = _counter(nets[0])
    nets[0].train_fused(mems[0], nsteps=2)
    assert _counter(nets[0]) == c0 + 2
    assert (nets[0].last_taus()[:, :B * N] == IQ.tau_draw(nets[0].tau_seed, c0 + 1, 2, B, N)).all()
    assert (IQ.tau_draw(nets[0].tau_seed, c0, 2, B, N) != IQ.tau_draw(nets[0].tau_seed, c0 + 1, 2, B, N)).any()
    random.seed(5)
    mems[1].seed_device_rng(random)
    for _ in range(2):
        nets[1].train(mems[1].getMinibatch())
    assert _counter(nets[1]) == c0 + 2
    for x, y in zip(nets[0].get_weights(with_states=False), nets[1].get_weights(with_states=False)):
        assert (x == y).all()
    assert (nets[0].last_costs(2) == nets[1].last_costs(2)).all()


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("K", [1, 32])
def test_predict_paths_agree(mode, K):
    """Host predict, predict_device and the captured fast path of three twins (same weights, same counter) agree bit
    for bit; padding rows come back as exact zeros; Q is the mean over the K rows of the generator's draw; the next
    predict draws fresh tau.  With every fc2 row equal all Q tie, and the agent's argmax takes action 0."""
    import ctypes as C
    from simple_dqn_b200 import StateBuffer, Stream, _lib as L
    B, A = 32, 6
    stream = Stream()
    nets = [_inet(A, 8, K, B, stream=stream, mode=mode) for _ in range(3)]
    sb = StateBuffer(make_args(), stream=stream)
    rs = np.random.RandomState(1)
    for _ in range(4):
        sb.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    ds = sb.getStateMinibatch()
    c0 = _counter(nets[0])
    fast = nets[0].predict(ds)
    host = nets[1].predict(np.asarray(ds))
    qp = nets[2].device_view(L.NET_PTR_Q_ONLINE, (B, A)).ptr
    L.call("b200dqn_net_predict_device", nets[2]._h, C.c_void_p(ds.device_ptr()), 1, C.c_void_p(qp), nets[2]._stream)
    dev = nets[2]._read_f32(L.NET_PTR_Q_ONLINE, (B, A))
    assert (fast[0] == host[0]).all() and (dev[0] == host[0]).all()
    assert (fast[1:] == 0).all() and (dev[1:] == 0).all() and (host[0] != 0).any()
    for net in nets:
        assert _counter(net) == c0 + 1
    assert (nets[1].last_taus()[0, :B * K] == IQ.tau_draw(nets[1].tau_seed, c0, 1, B, K)[0]).all()
    assert (host == IQ.q_values(nets[1].last_iqn_quantiles()[0, :B * K], K)).all()
    fast2 = nets[0].predict(ds)             # the captured graph again: the counter moves on the device
    assert _counter(nets[0]) == c0 + 2 and not (fast2[0] == fast[0]).all()
    ws, ss = nets[0].get_weights()
    ws[4][:] = ws[4][:1]
    nets[0].set_weights(ws, ss)
    q = nets[0].predict(ds)
    assert (q[0] == q[0][0]).all() and int(np.argmax(q[0])) == 0


@pytest.mark.parametrize("mode", ENGINES)
def test_train_paths_agree(mode):
    """train_fused, sample + train_sampled_cost, step_host and sample + gather + train_device of four twins on four
    equal rings give the same weights, states and costs, bit for bit."""
    import ctypes as C
    import random
    from simple_dqn_b200 import DeviceMinibatch, Stream, _lib as L
    B, A, N = 8, 4, 8
    out = []
    for path in ("fused", "sampled", "step_host", "device"):
        stream = Stream()
        ring, mem = _ring_pair(batch=B, stream=stream)
        net = _inet(A, N, 32, B, stream=stream, mode=mode)
        random.seed(9)
        mem.seed_device_rng(random)
        for _ in range(2):
            if path == "fused":
                net.train_fused(mem, 1)
            elif path == "sampled":
                mem.sample()
                cost = C.c_float()
                L.call("b200dqn_net_train_sampled_cost", net._h, mem._h, C.byref(cost), net._stream)
            elif path == "step_host":
                L.call("b200dqn_net_step_host", net._h, mem._h, 0, None, None, None, None, 1, None, 0, None, None,
                       net._stream)
            else:
                mem.sample()
                L.call("b200dqn_replay_gather", mem._h, mem._stream)
                ptr = lambda which: C.c_void_p(mem.device_view(which, np.uint8, (1,)).ptr)
                L.call("b200dqn_net_train_device", net._h, ptr(L.PTR_PRESTATES), ptr(L.PTR_MB_ACTIONS),
                       ptr(L.PTR_MB_REWARDS), ptr(L.PTR_POSTSTATES), ptr(L.PTR_MB_TERMINALS), net._stream)
        out.append((net.last_costs(2), net.get_weights(with_states=False), net.get_states(), _counter(net)))
    for o in out[1:]:
        assert (o[0] == out[0][0]).all() and o[3] == out[0][3]
        for x, y in zip(o[1], out[0][1]):
            assert (x == y).all()
        for x, y in zip(o[2], out[0][2]):
            for p, q in zip(x, y):
                assert (p == q).all()


def test_checkpoints_target_sync_and_refusals(tmp_path):
    from simple_dqn_b200 import DeepQNetwork
    net = _inet(4, 8, 32, 4)
    net.train(random_minibatch(4, 4, seed=1))
    for layout in ("neon-1.3.0", "pre-1.0"):
        path = str(tmp_path / ("iqn_%s.pkl" % layout))
        net.save_weights(path, layout=layout)
        twin = _inet(4, 8, 32, 4, seed=9)
        twin.load_weights(path)
        for x, y in zip(net.get_weights(with_states=False), twin.get_weights(with_states=False)):
            assert (x == y).all()
        for x, y in zip(net.get_states(), twin.get_states()):
            for p, q in zip(x, y):
                assert (p == q).all()
        plain = DeepQNetwork(4, make_args(batch_size=4), math_mode="fp32")
        with pytest.raises(AssertionError, match="five"):
            plain.load_weights(path)
    plain.save_weights(str(tmp_path / "plain.pkl"))
    with pytest.raises(AssertionError, match="six"):
        net.load_weights(str(tmp_path / "plain.pkl"))
    net.update_target_network()
    for x, y in zip(net.get_weights(0, with_states=False), net.get_weights(1, with_states=False)):
        assert (x == y).all()
    with pytest.raises(NotImplementedError):
        net.set_double_dqn(True)
    with pytest.raises(NotImplementedError):
        net.comm_init(DeepQNetwork.comm_unique_id(), 0, 1)
    from simple_dqn_b200 import _lib as L
    with pytest.raises(AssertionError):
        net.device_view(L.NET_PTR_QUANTILES, (1,))
    with pytest.raises(AssertionError):
        plain.device_view(L.NET_PTR_IQN_TAUS, (1,))
    with pytest.raises(AssertionError):   # layer 5 exists on an IQN net only
        L.call("b200dqn_net_layer_shape", plain._h, 5, None, None)


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
def test_launch_count_and_trajectory(mode, sched):
    """The captured step's launch count equals the static one; five host steps stay within the trajectory bars of the
    numpy IQN step driven by the device's taus."""
    import random
    from simple_dqn_b200 import Stream
    stream = Stream() if sched == "branches" else None
    B, A, N = 8, 4, 8
    from simple_dqn_b200 import DeepQNetwork
    net = _inet(A, N, 32, B, stream=stream, mode=mode)
    plain = DeepQNetwork(A, make_args(batch_size=B), math_mode=mode, stream=stream)
    # the tau draw, the embedding, the modulation, its backward and dWe, k_fc2_dist and, on the SIMT engine, fc2's own
    # gradient kernel (the tensor-core engine updates fc2 in a kernel of its own already)
    extra = 7 if mode == "fp32" else 6
    assert net.launches_per_step() == plain.launches_per_step() + extra
    if stream is not None:   # the captured graphs count their launches
        counts = []
        for n in (plain, _inet(A, N, 32, B, stream=stream, mode=mode)):
            ring, mem = _ring_pair(batch=B, stream=stream)
            random.seed(3)
            mem.seed_device_rng(random)
            n.train_fused(mem, nsteps=1)
            counts.append(n.launches_per_step())
        assert counts[1] == counts[0] + extra, counts
    ws = [w.astype(F32).copy() for w in net.get_weights()[0]]
    ss = [s[0].copy() for s in net.get_states()]
    tws = net.get_weights(which=1, with_states=False)
    w0 = [w.copy() for w in ws]
    for step in range(5):
        mb = random_minibatch(B, A, seed=40 + step)
        net.train(mb)
        taus = net.last_taus()[:, :B * N]
        IQ.numpy_step(ws, ss, tws, mb, taus, 1.0)
    w1 = net.get_weights(with_states=False)
    for layer in range(6):
        assert rel_l2(w1[layer] - w0[layer], ws[layer] - w0[layer]) <= 2e-2, layer
