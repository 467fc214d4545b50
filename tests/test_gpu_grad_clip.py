"""Global gradient-norm clipping on the device against tests/grad_clip_oracle.py: every S_l against an exactly rounded
sum over the device's own get_grads(), N and c32 bit for bit from the device's S, and every weight and optimizer state
of layers 0-5 bit for bit equal to the oracle's update on gg' (batch size 1), under every head (plus a soft target
update on top), both engines, both schedules and all three optimizers; the FQF fraction layer exactly as unclipped.  A
twin loaded with the weights takes the same next step (so the tensor-core images equal a fresh pack) at every batch-size
dispatch and history length 1 and 16; every train entry point clips; a net whose norm never reaches M trains bit for bit
like an unclipped one; the launch count; the refusals."""
import ctypes as C
import random

import numpy as np
import pytest

import grad_clip_oracle as CLIP
import soft_target_oracle as SOFT
from oracle import dqn_oracle as O
from test_gpu_distributional import _L, _ring_pair
from test_gpu_soft_target import HEADS, _bits, _snet

pytestmark = pytest.mark.gpu

F32 = np.float32
MODES = ["tcgen05", "fp32"]
M_SMALL = 1e-5   # far below the norm of any step here: c32 < 1 is asserted
CHEADS = dict(HEADS, soft={})


def _cnet(mode, head="scalar", stream=None, max_grad_norm=M_SMALL, **kw):
    tau = 0.005 if head == "soft" else 0.0
    return _snet(mode, tau, stream=stream, max_grad_norm=max_grad_norm, **dict(CHEADS[head], **kw))


def _snapshot(net, which=0):
    ws, _ = net.get_weights(which=which)
    return [w.copy() for w in ws], [[p.copy() for p in s] for s in net.get_states(which=which)]


def _oracle_update(optimizer, ws, ss, grads, bsz, t, lr=0.00025):
    if optimizer == "rmsprop":
        O.rmsprop_update(ws, [s[0] for s in ss], grads, bsz, lr=lr)
    elif optimizer == "adam":
        O.adam_update(ws, ss, grads, bsz, t, lr=lr)
    else:
        O.adadelta_update(ws, ss, grads, bsz)


def _check_step(net, before, optimizer="rmsprop", t=1, max_grad_norm=M_SMALL):
    """The step just taken is the rule on the device's own gradients: S_l, N, c32, and layers 0-5 bit for bit."""
    w0, s0 = before
    nl = 6 if len(w0) > 5 else 5
    g = net.get_grads()
    sq = net.last_grad_sq()
    gg = CLIP.scaled_grads(g[:nl], net.batch_size)
    for l in range(nl):
        exact = CLIP.layer_sq(gg[l])
        assert abs(sq[l] - exact) <= (gg[l].size - 1) * 2.0 ** -53 * exact, (l, sq[l], exact)
    assert (sq[nl:] == 0).all()
    n = net.last_grad_norm()
    assert n == CLIP.norm_from_sq(sq)
    c = net.last_clip_scale()
    assert c == CLIP.clip_scale(n, max_grad_norm)
    if max_grad_norm == M_SMALL:
        assert c < 1
    ggp = [(x * c).astype(F32) for x in gg]
    ws, ss = [w.copy() for w in w0[:nl]], [[p.copy() for p in s] for s in s0[:nl]]
    _oracle_update(optimizer, ws, ss, ggp, 1, t)
    got_w, got_s = net.get_weights(with_states=False), net.get_states()
    for l in range(nl):
        assert (_bits(got_w[l]) == _bits(ws[l])).all(), l
        for k, (a, b) in enumerate(zip(got_s[l], ss[l])):
            assert (_bits(a) == _bits(b)).all(), (l, k)


def _mems(head, stream, batch=32, hist=4):
    per = head == "per_nstep"
    _, mem = _ring_pair(batch=batch, hist=hist, stream=stream, prioritized_replay=per, beta0=0.4)
    if per:
        mem.set_n_step(3)
    return mem


def _train_sampled(net, mem, seed, batch=32):
    from simple_dqn_b200 import DeviceMinibatch
    mem.set_indexes(np.array(random.Random(seed).sample(range(50, 2900), batch), np.int32))
    net.train(DeviceMinibatch(mem, sampled=True))


@pytest.mark.parametrize("optimizer", ["rmsprop", "adam", "adadelta"])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("sched", ["branches", "serial"])
@pytest.mark.parametrize("head", sorted(CHEADS))
def test_one_step_follows_the_rule(optimizer, mode, sched, head):
    from simple_dqn_b200 import Stream
    stream = Stream() if sched == "branches" else None
    mem = _mems(head, stream)
    net = _cnet(mode, head, stream=stream, optimizer=optimizer)
    assert net.max_grad_norm == M_SMALL
    before = _snapshot(net)
    tw = net.get_weights(which=1, with_states=False)
    twin = None
    if head == "fqf":   # the fraction layer trains exactly as on an unclipped net
        twin = _cnet(mode, head, stream=stream, optimizer=optimizer, max_grad_norm=0.0)
        assert twin.max_grad_norm is None
        _train_sampled(twin, mem, 0)
    _train_sampled(net, mem, 0)
    _check_step(net, before, optimizer)
    if twin is not None:
        assert (_bits(net.get_weights(with_states=False)[6]) == _bits(twin.get_weights(with_states=False)[6])).all()
        for a, b in zip(net.get_states()[6], twin.get_states()[6]):
            assert (_bits(a) == _bits(b)).all()
    if head == "soft":   # the blend follows the clipped update
        for got, exp in zip(net.get_weights(which=1, with_states=False),
                            SOFT.blend_layers(tw, net.get_weights(with_states=False), 0.005)):
            assert (_bits(got) == _bits(exp)).all()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("batch,hist", [(1, 4), (32, 1), (33, 4), (256, 16), (257, 4)])
@pytest.mark.parametrize("head", ["scalar", "dueling", "c51"])
def test_twin_loaded_with_the_clipped_weights_takes_the_same_step(mode, batch, hist, head):
    """Two clipped steps, then a clipped twin loaded with the weights and states takes the next step bit for bit like
    the first net (the tensor-core tile images after a clipped update equal a fresh pack), and that step follows the
    rule too."""
    from simple_dqn_b200 import Stream
    stream, tstream = Stream(), Stream()
    _, mem = _ring_pair(batch=batch, hist=hist, stream=stream)
    _, tmem = _ring_pair(batch=batch, hist=hist, stream=tstream)
    kw = dict(batch=batch, hist=hist)
    net = _cnet(mode, head, stream=stream, **kw)
    for step in range(2):
        _train_sampled(net, mem, step, batch)
    twin = _cnet(mode, head, stream=tstream, seed=11, **kw)
    for which in (0, 1):
        twin.set_weights(net.get_weights(which=which, with_states=False), net.get_states(which=which), which=which)
    before = _snapshot(net)
    _train_sampled(net, mem, 9, batch)
    _train_sampled(twin, tmem, 9, batch)
    _check_step(net, before)
    assert (_bits(net.last_costs(1)) == _bits(twin.last_costs(1))).all()
    for a, b in zip(net.last_q(), twin.last_q()):
        assert (_bits(a) == _bits(b)).all()
    for a, b in zip(net.get_weights(with_states=False), twin.get_weights(with_states=False)):
        assert (_bits(a) == _bits(b)).all()
    assert (net.last_grad_sq().view(np.uint64) == twin.last_grad_sq().view(np.uint64)).all()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("entry", ["host_tuple", "train_device", "sampled", "unsampled", "fused", "fused_replay",
                                   "step_host"])
def test_every_train_entry_point_clips(mode, entry):
    from helpers import random_minibatch
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    _, mem = _ring_pair(stream=stream)
    random.seed(5)
    mem.seed_device_rng(random)
    net = _cnet(mode, stream=stream)
    if entry == "fused_replay":   # the last of three steps of one captured graph, replayed
        net.train_fused(mem, 2)
    before = _snapshot(net)
    if entry == "host_tuple":
        net.train(random_minibatch(32, 4, 5))
    elif entry == "train_device":
        L = _L()
        mem.sample()
        L.call("b200dqn_replay_gather", mem._h, mem._stream)
        ptr = lambda which: C.c_void_p(mem.device_view(which, np.uint8, (1,)).ptr)
        L.call("b200dqn_net_train_device", net._h, ptr(L.PTR_PRESTATES), ptr(L.PTR_MB_ACTIONS),
               ptr(L.PTR_MB_REWARDS), ptr(L.PTR_POSTSTATES), ptr(L.PTR_MB_TERMINALS), net._stream)
    elif entry == "sampled":
        _train_sampled(net, mem, 3)
    elif entry == "unsampled":
        net.train(DeviceMinibatch(mem, sampled=False))
    elif entry in ("fused", "fused_replay"):
        net.train_fused(mem, 1)
    else:
        empty = np.zeros((0,) + tuple(mem.dims), np.uint8)
        net.step_host(mem, np.zeros(0, np.uint8), np.zeros(0, np.int64), empty, np.zeros(0, np.uint8), train_repeat=1)
    _check_step(net, before)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("head", ["scalar", "iqn"])
def test_a_norm_below_max_trains_bit_for_bit_like_no_clipping(mode, head):
    """M = 1e30: c32 = 1 at every step, and cost, weights, states and target equal an unclipped net's bit for bit."""
    from simple_dqn_b200 import Stream
    out = []
    for m in (1e30, 0.0):
        stream = Stream()
        _, mem = _ring_pair(stream=stream)
        random.seed(6)
        mem.seed_device_rng(random)
        net = _cnet(mode, head, stream=stream, max_grad_norm=m)
        net.train_fused(mem, 4)
        if m:
            assert net.last_clip_scale() == F32(1.0) and net.last_grad_norm() > 0
        out.append((net.last_costs(4), _snapshot(net), _snapshot(net, which=1)))
    (ca, (wa, sa), (ta, _)), (cb, (wb, sb), (tb, _)) = out
    assert (_bits(ca) == _bits(cb)).all()
    for x, y in zip(wa + ta, wb + tb):
        assert (_bits(x) == _bits(y)).all()
    for x, y in zip(sa, sb):
        for p, q in zip(x, y):
            assert (_bits(p) == _bits(q)).all()


@pytest.mark.parametrize("mode", MODES)
def test_two_identical_nets_give_identical_sums(mode):
    from simple_dqn_b200 import Stream
    sums = []
    for _ in range(2):
        stream = Stream()
        _, mem = _ring_pair(stream=stream)
        random.seed(7)
        mem.seed_device_rng(random)
        net = _cnet(mode, "iqn", stream=stream)
        net.train_fused(mem, 3)
        sums.append((net.last_grad_sq().view(np.uint64).copy(), net.last_clip_scale()))
    assert (sums[0][0] == sums[1][0]).all() and sums[0][1] == sums[1][1]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("head", ["scalar", "c51", "iqn", "fqf"])
def test_launch_count_grows_by_the_documented_launches(mode, head):
    """Tensor-core engine 15 (3 conv reduces, 5 sums of squares, clip_scale, fc2's reduce and update split in two, and
    5 conv image packs beside the 3 conv updates); SIMT engine 12 with the scalar fc2 (5 reduces, 5 sums of squares,
    clip_scale, fc1 and fc2 updated apart), 11 with a per-action fc2; an embedding adds its sum of squares and its
    update.  In the static count and in the count taken while the step graph is captured."""
    from simple_dqn_b200 import Stream
    stream = Stream()
    _, mem = _ring_pair(stream=stream)
    random.seed(1)
    mem.seed_device_rng(random)
    extra = (15 if mode == "tcgen05" else 12 if head == "scalar" else 11) + (2 if head in ("iqn", "fqf") else 0)
    static, captured = [], []
    for m in (0.0, 10.0):
        net = _cnet(mode, head, stream=stream, max_grad_norm=m)
        static.append(net.launches_per_step())
        net.train_fused(mem, 1)
        captured.append(net.launches_per_step())
    assert static[1] - static[0] == extra, static
    assert captured[1] - captured[0] == extra, captured


def test_selectors_are_einval_without_clipping_and_comm_init_refuses():
    net = _cnet("tcgen05", max_grad_norm=0.0)
    L = _L()
    for which in (L.NET_PTR_GRAD_SQ, L.NET_PTR_GRAD_NORM, L.NET_PTR_CLIP_SCALE):
        p, b = C.c_void_p(), C.c_size_t()
        with pytest.raises(AssertionError, match="gradient-norm"):
            L.call("b200dqn_net_device_ptr", net._h, which, C.byref(p), C.byref(b))
    with pytest.raises(ValueError):
        net.last_grad_norm()
    clipped = _cnet("tcgen05", max_grad_norm=10.0)
    with pytest.raises(NotImplementedError, match="gradient-norm"):
        clipped.comm_init(bytes(128), 0, 2)
