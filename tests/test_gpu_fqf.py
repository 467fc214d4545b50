"""The fully parameterized quantile function head (FQF) on the device against tests/fqf_oracle.py and
tests/iqn_oracle.py, each stage fed the device's own inputs so that errors do not carry over: the logits bit for bit;
the proposal q, tau and tauhat within one fp32 ulp (the device's exp); the cosine features within one ulp; and bit for
bit phi, X, theta, Q, T, the row costs, the cost, dtheta, dZ4 and its fp16 planes, fc2's gradient, g, dl, dW_f, dWe and
the updates of layers 4-6.  fc1's forward, dgrad and wgrad and conv3's wgrad are held to the float64 bounds of
tests/kernel_ref.py, and the boundary quantiles to a float64 recomputation.  Both engines and both schedules, RMSProp,
Adam and Adadelta, kappa 0, 0.5 and 1, first-index ties of a*, target_steps = 0, 4096 rows, a prioritized ring with
n-step returns and random shifts; every train path against the others, the predict paths, the initial proposal,
checkpoints, the target sync, the refusals and the launch count."""
import numpy as np
import pytest

import c51_oracle as C51
import fqf_oracle as FQ
import iqn_oracle as IQ
import kernel_ref as K
from helpers import make_args, random_minibatch, rel_l2
from test_gpu_distributional import _gather, _optimize, _ring_pair
from test_gpu_kernels import _chain, _check

pytestmark = pytest.mark.gpu

F32 = np.float32
# fc1's input column n in Neon's (c, p, q) order sits at internal column (p * 7 + q) * 64 + c
PERM = np.array([((n // 7 % 7) * 7 + n % 7) * 64 + n // 49 for n in range(3136)])
FLR = 1e-3   # a fraction learning rate large enough to move W_f visibly in two steps


def _fnet(A=4, N=8, batch=8, kappa=1.0, stream=None, optimizer="rmsprop", target_steps=10000, seed=3, mode="fp32",
          tie=False, **kw):
    """tie: the target network's fc2 rows are all equal, so every target Q of a sample ties and a* must be action 0."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, random_seed=seed, fqf=True, num_fractions=N, fraction_lr=FLR,
                                    clip_error=kappa, optimizer=optimizer, target_steps=target_steps, **kw),
                       math_mode=mode, stream=stream)
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


def _internal(wf_neon):
    """(N, 3136) Neon fraction layer -> fc1's internal column order."""
    out = np.empty_like(wf_neon)
    out[:, PERM] = wf_neon
    return out


def _we_internal(we_neon):
    out = np.empty((64, 3136), F32)
    out[:, PERM] = we_neon.T
    return out


def _ulp_close(dev, ref):
    ref = np.asarray(ref, F32)
    return (np.abs(dev.astype(np.float64) - ref.astype(np.float64)) <= np.spacing(np.abs(ref))).all()


def _states(net):
    return [[a.copy() for a in s] for s in net.get_states()]


def _check_step(net, before, tws, actions, returns, kappa, w=None, t=1):
    """Every stage of the last train step.  before: (weights, states) of the online net ahead of the step; tws the
    target weights; returns per-sample (R, g)."""
    from simple_dqn_b200 import _lib as L
    A, N, B = net.num_actions, net.num_fractions, net.batch_size
    R = ld = B * N
    ws, ss = before
    h3 = _read(net, L.NET_PTR_H3, (B, 3136))
    l = net.last_fraction_logits()
    assert (l == FQ.logits(h3, _internal(ws[6]))).all()
    q, frac = net.last_fraction_probs(), net.last_fractions()
    eq, etau, etauhat = FQ.proposal(l)
    assert _ulp_close(q, eq) and _ulp_close(frac, etau)
    assert (frac[:, 0] == 0).all() and (frac[:, -1] == 1).all()
    tau = net.last_taus()[:, :R]
    assert _ulp_close(tau[0], etauhat.reshape(-1)) and (tau[1] == tau[0]).all()
    c = _read(net, L.NET_PTR_IQN_COS, (2, ld, 64))
    ref = np.cos((np.pi * np.arange(64)) * tau[:, :, None].astype(np.float64))
    assert (np.abs(c - ref) <= np.spacing(np.abs(ref).astype(F32))).all()
    phi = _read(net, L.NET_PTR_IQN_PHI, (2, ld, 3136))
    for z, wz in ((0, ws), (1, tws)):
        assert (phi[z] == IQ.phi(c[z], _we_internal(wz[5]))).all(), z
    x = _read(net, L.NET_PTR_IQN_X, (2, ld, 3136))
    assert (x[0] == IQ.modulate(h3, phi[0], N)).all()
    mode = net.math_mode
    h4 = _read(net, L.NET_PTR_H4, (ld, 512))
    xn = x[0][:, PERM]
    ratios = _check("fc1_fwd", mode, K.fc_fwd, xn, ws[3], h4, _chain(mode, "fc1_fwd", R, 4), post=K.relu)
    theta = net.last_iqn_quantiles()
    assert (theta[0] == IQ.logits(h4, ws[4].T)).all()
    q0, q1, astar, T, loss, g = FQ.head(theta, tau[0], frac, actions, returns, kappa, w)
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
    # the boundary pass: the online network at tau_1..tau_{N-1}, against a float64 recomputation
    bnd = net.last_boundary_quantiles()
    btau = frac[:, 1:-1].reshape(-1).astype(np.float64)
    bc = np.cos((np.pi * np.arange(64)) * btau[:, None])
    bphi = np.maximum(bc @ ws[5].T.astype(np.float64), 0)
    bx = np.repeat(h3.astype(np.float64), N - 1, axis=0)[:, PERM] * bphi
    bh4 = np.maximum(bx @ ws[3].T.astype(np.float64), 0)
    assert rel_l2(bnd.reshape(-1, A), bh4 @ ws[4].T.astype(np.float64)) <= 1e-4
    acts = np.asarray(actions, np.int64)
    theta_a = theta[0, :R].reshape(B, N, A)[np.arange(B), :, acts]
    beta = bnd[np.arange(B), :, acts]
    eg, edl = FQ.fraction_grads(theta_a, beta, q, w)
    assert (net.last_fraction_grads() == eg).all()
    dl = net.last_fraction_logit_grads()
    assert (dl == edl).all()
    dz4 = _read(net, L.NET_PTR_DZ4, (ld, 512))
    assert (dz4 == IQ.dz4(h4, ws[4].T, actions, g, N)).all()
    if mode == "tcgen05":   # the planes the tensor-core fc1 dgrad and wgrad read
        import ctypes as C
        p, b = C.c_void_p(), C.c_size_t()
        L.call("b200dqn_net_device_ptr", net._h, L.NET_PTR_DZ4_PLANES, C.byref(p), C.byref(b))
        lo_off = b.value // 2 - B * 512
        hi16 = L.download(net.device, p.value, (R, 512), np.float16, net._stream)
        lo16 = L.download(net.device, p.value + 2 * lo_off, (R, 512), np.float16, net._stream)
        ehi, elo = C51.fp16_planes(dz4)
        assert (hi16.view(np.uint16) == ehi.view(np.uint16)).all() and (lo16.view(np.uint16) == elo.view(np.uint16)).all()
    grads = net.get_grads()
    assert len(grads) == 7
    assert (grads[4] == IQ.fc2_grad(h4, actions, g, N, A)).all()
    dx = _read(net, L.NET_PTR_IQN_DX, (ld, 3136))
    ratios.update(_check("fc1_dgrad", mode, K.fc_dgrad, dz4, ws[3], dx[:, PERM], _chain(mode, "fc1_dgrad", R, 4),
                         mask=xn > 0))
    nw = _chain(mode, "fc1_wgrad", min(R, 256), 4) + -(-R // 256) if mode == "tcgen05" else R
    ratios.update(_check("fc1_wgrad", mode, K.fc_wgrad, xn, dz4, grads[3], nw))
    dpsi, dphi = IQ.mod_bwd(dx, phi[0], h3, N)
    assert (_read(net, L.NET_PTR_DZ3, (B, 3136)) == dpsi).all()
    h2 = net.last_activations()[1]
    ratios.update(_check("conv3_wgrad", mode, K.conv_wgrad(2), h2, dpsi.reshape(B, 7, 7, 64).transpose(0, 3, 1, 2),
                         grads[2], _chain(mode, "conv3_wgrad", B, 4)))
    # The SIMT fc1 wgrad (the IQN head's kernel, unchanged) sums all nb N rows in one fp32 chain.  At the first proposal
    # every sample has the same tauhat, so the rows are strongly correlated and the rounding errors do not cancel as the
    # sqrt(n) bound assumes: at 1024 rows it measured 1.13 times that bound on an H100.
    wgrad_cap = 1.5 if mode == "fp32" and R > 256 else 1.0
    assert ratios.pop("fc1_wgrad") <= wgrad_cap, ratios
    assert max(ratios.values()) <= 1.0, ratios
    assert (_read(net, L.NET_PTR_IQN_DPHI, (ld, 3136)) == dphi).all()
    assert (grads[5] == IQ.we_grad(c[0], dphi)[:, PERM].T).all()
    assert (grads[6] == FQ.wf_grad(dl, h3)[:, PERM]).all()
    w1, s1 = net.get_weights()[0], net.get_states()
    for layer in (4, 5, 6):
        ew, es = _optimize_lr(net.optimizer, ws[layer], ss[layer], grads[layer], B, t, FLR if layer == 6 else 0.00025)
        assert (w1[layer] == ew).all(), layer
        for p_, q_ in zip(s1[layer], es):
            assert (p_ == q_).all(), layer
    return astar


def _optimize_lr(optimizer, w, states, g, batch, t, lr):
    from oracle import dqn_oracle as O
    if optimizer == "adadelta":
        return _optimize(optimizer, w, states, g, batch, t)
    w = w.copy()
    states = [s.copy() for s in states]
    if optimizer == "rmsprop":
        O.rmsprop_update([w], [states[0]], [g], batch, lr=lr)
    else:
        O.adam_update([w], [states[:2]], [g], batch, t, lr=lr)
    return w, states


ENGINES = ["tcgen05", "fp32"]
STEP = [  # (batch, A, N, kappa, optimizer, target_steps, tie)
    (8, 4, 8, 1.0, "rmsprop", 10000, False), (1, 1, 2, 1.0, "rmsprop", 10000, False),
    (5, 2, 64, 0.0, "adam", 10000, True), (32, 18, 32, 0.5, "adadelta", 0, False),
    (64, 32, 64, 1.0, "rmsprop", 10000, False), (65, 4, 8, 1.0, "adam", 10000, False),
]


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
@pytest.mark.parametrize("batch,A,N,kappa,optimizer,ts,tie", STEP)
def test_train_step_stages(mode, sched, batch, A, N, kappa, optimizer, ts, tie):
    from simple_dqn_b200 import Stream
    stream = Stream() if sched == "branches" else None
    net = _fnet(A, N, batch, kappa, stream, optimizer, ts, mode=mode, tie=tie)
    assert net.layer_shapes()[5:] == [(3136, 64), (N, 3136)]
    for step in range(2):
        pre, act, rew, post, term = random_minibatch(batch, A, seed=10 + step)
        before = (net.get_weights()[0], _states(net))
        tws = net.get_weights(which=1, with_states=False) if ts else before[0]
        net.train((pre, act, rew, post, term))
        if step == 0:   # W_f starts at zero: the first proposal is the quantile-regression head's midpoints
            assert (net.last_taus()[0, :batch * N] == np.tile(FQ.midpoints(N), batch)).all()
        returns = [IQ.one_step_return(rew[i], term[i], 0.99) for i in range(batch)]
        astar = _check_step(net, before, tws, act, returns, kappa, t=step + 1)
        if tie:
            assert (astar == 0).all()
    assert (net.get_weights()[0][6] != 0).any()


@pytest.mark.parametrize("mode", ENGINES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
def test_weighted_nstep_shifted_step_stages(mode, sched):
    """A step on a prioritized ring with n-step 3 and random_shift 4: the importance weights scale dtheta and g, the
    priority is the unweighted row loss, and every other stage holds bit for bit."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    import random
    stream = Stream() if sched == "branches" else None
    B, A, N = 16, 4, 8
    ring, mem = _ring_pair(batch=B, stream=stream, prioritized_replay=True, beta0=0.4, terminal_p=0.1)
    mem.set_n_step(3)
    net = _fnet(A, N, B, 1.0, stream, mode=mode, random_shift=4)
    idx0 = np.array(random.Random(0).sample(range(4, 2990), B), np.int32)
    for step in range(2):
        mem.set_indexes(np.roll(idx0, step))
        before = (net.get_weights()[0], _states(net))
        tws = net.get_weights(which=1, with_states=False)
        net.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, np.roll(idx0, step), 3)
        w = mem.last_weights
        returns = [IQ.n_step_return(mb[2][i], mb[4][i], 0.99) for i in range(B)]
        _check_step(net, before, tws, mb[1].astype(np.int64), returns, 1.0, w=w, t=step + 1)
        if step:
            assert (w != F32(1)).any()


@pytest.mark.parametrize("mode", ENGINES)
def test_train_paths_agree(mode):
    """train_fused, sample + train_sampled_cost, step_host and the host tuple of four twins on four equal rings give
    the same weights (all seven layers), states and costs, bit for bit."""
    import ctypes as C
    import random
    from simple_dqn_b200 import Stream, _lib as L
    B, A, N = 8, 4, 8
    out = []
    for path in ("fused", "sampled", "step_host", "host"):
        stream = Stream()
        ring, mem = _ring_pair(batch=B, stream=stream)
        net = _fnet(A, N, B, stream=stream, mode=mode)
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
        out.append((net.last_costs(2), net.get_weights(with_states=False), net.get_states()))
    for o in out[1:]:
        assert (o[0] == out[0][0]).all()
        for x, y in zip(o[1], out[0][1]):
            assert (x == y).all()
        for x, y in zip(o[2], out[0][2]):
            for p, q in zip(x, y):
                assert (p == q).all()


@pytest.mark.parametrize("mode", ENGINES)
def test_predict_paths_agree(mode):
    """Host predict, predict_device and the captured fast path of three twins with a trained W_f agree bit for bit;
    padding rows come back as exact zeros; Q follows rule 4 on the device's fractions and quantiles."""
    import ctypes as C
    from simple_dqn_b200 import StateBuffer, Stream, _lib as L
    B, A, N = 32, 6, 8
    stream = Stream()
    nets = [_fnet(A, N, B, stream=stream, mode=mode) for _ in range(3)]
    rs = np.random.RandomState(2)
    wf = (rs.randn(N, 3136) * 0.01).astype(F32)
    for net in nets:
        ws, ss = net.get_weights()
        ws[6] = wf
        net.set_weights(ws, ss)
    sb = StateBuffer(make_args(), stream=stream)
    for _ in range(4):
        sb.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    ds = sb.getStateMinibatch()
    fast = nets[0].predict(ds)
    host = nets[1].predict(np.asarray(ds))
    qp = nets[2].device_view(L.NET_PTR_Q_ONLINE, (B, A)).ptr
    L.call("b200dqn_net_predict_device", nets[2]._h, C.c_void_p(ds.device_ptr()), 1, C.c_void_p(qp), nets[2]._stream)
    dev = nets[2]._read_f32(L.NET_PTR_Q_ONLINE, (B, A))
    assert (fast[0] == host[0]).all() and (dev[0] == host[0]).all()
    assert (fast[1:] == 0).all() and (dev[1:] == 0).all() and (host[0] != 0).any()
    frac = nets[1].last_fractions()
    assert not (frac[0] == np.linspace(0, 1, N + 1)).all()
    assert (host == FQ.q_values(nets[1].last_iqn_quantiles()[0], frac)).all()
    assert (nets[0].predict(ds)[0] == fast[0]).all()   # no draw: the same states give the same Q


def test_initial_weights_checkpoints_target_sync_and_refusals(tmp_path):
    from simple_dqn_b200 import DeepQNetwork, _lib as L
    net = _fnet(4, 8, 4)
    iqn = DeepQNetwork(4, make_args(batch_size=4, random_seed=3, implicit_quantiles=True, num_tau_samples=8),
                       math_mode="fp32")
    fresh = DeepQNetwork(4, make_args(batch_size=4, random_seed=3, fqf=True, num_fractions=8), math_mode="fp32")
    assert fresh.fraction_lr == 2.5e-9
    for which in (0, 1):   # layers 0-5 are drawn as on an IQN net of the same seed; W_f starts at zero
        a, b = fresh.get_weights(which, with_states=False), iqn.get_weights(which, with_states=False)
        for x, y in zip(a[:6], b):
            assert (x == y).all()
        assert a[6].shape == (8, 3136) and (a[6] == 0).all()
    net.train(random_minibatch(4, 4, seed=1))
    for layout in ("neon-1.3.0", "pre-1.0"):
        path = str(tmp_path / ("fqf_%s.pkl" % layout))
        net.save_weights(path, layout=layout)
        twin = _fnet(4, 8, 4, seed=9)
        twin.load_weights(path)
        for x, y in zip(net.get_weights(with_states=False), twin.get_weights(with_states=False)):
            assert (x == y).all()
        for x, y in zip(net.get_states(), twin.get_states()):
            for p, q in zip(x, y):
                assert (p == q).all()
        with pytest.raises(AssertionError, match="six"):
            iqn.load_weights(path)
    for other in (iqn, DeepQNetwork(4, make_args(batch_size=4), math_mode="fp32")):
        path = str(tmp_path / "other.pkl")
        other.save_weights(path)
        with pytest.raises(AssertionError, match="seven"):
            net.load_weights(path)
    net.update_target_network()
    for x, y in zip(net.get_weights(0, with_states=False), net.get_weights(1, with_states=False)):
        assert (x == y).all()
    for x, y in zip(net.get_states(0), net.get_states(1)):
        for p, q in zip(x, y):
            assert (p == q).all()
    with pytest.raises(NotImplementedError):
        net.set_double_dqn(True)
    with pytest.raises(NotImplementedError):
        net.comm_init(DeepQNetwork.comm_unique_id(), 0, 1)
    with pytest.raises(AssertionError):
        net.device_view(L.NET_PTR_IQN_TAU_COUNTER, (1,))
    with pytest.raises(AssertionError):
        iqn.device_view(L.NET_PTR_FQF_LOGITS, (1,))
    for h in (iqn._h, DeepQNetwork(4, make_args(batch_size=4), math_mode="fp32")._h):   # layer 6: FQF nets only
        with pytest.raises(AssertionError):
            L.call("b200dqn_net_layer_shape", h, 6, None, None)
    with pytest.raises(AssertionError):
        L.call("b200dqn_net_layer_shape", net._h, 7, None, None)


@pytest.mark.parametrize("mode", ENGINES)
def test_launch_count(mode):
    """The captured step's launch count equals the static one: an FQF step launches five kernels more than an IQN
    step (the boundary pass's phi, modulation, fc1 and fc2, and dW_f), the proposal taking the tau draw's place."""
    import random
    from simple_dqn_b200 import DeepQNetwork, Stream
    stream = Stream()
    B, A, N = 8, 4, 8
    iqn = DeepQNetwork(A, make_args(batch_size=B, implicit_quantiles=True, num_tau_samples=N, num_quantile_samples=N),
                       math_mode=mode, stream=stream)
    net = _fnet(A, N, B, stream=stream, mode=mode)
    assert net.launches_per_step() == iqn.launches_per_step() + 5
    counts = []
    for n in (iqn, net):
        ring, mem = _ring_pair(batch=B, stream=stream)
        random.seed(3)
        mem.seed_device_rng(random)
        n.train_fused(mem, nsteps=1)
        counts.append(n.launches_per_step())
    assert counts[1] == counts[0] + 5, counts
