"""The train step at every value of the flags it turns into numbers, bit for bit wherever the device does scalar work.

The head (k_head) and the cost (k_cost_finish) at the reward bounds, discount rates and error clips of
test_oracle_flags.py, which ties the restatements used here to the reference.  Each case trains one step on a ring
whose rewards reach the int64 extremes, through train_fused (so the ring's int64 path is in the loop), on both
engines, with the vanilla target, the Double DQN target and a prioritized ring (beta0 = 0.4, weights not all 1).
The deltas, the row costs, the TD errors and the batch cost equal their restatement from the device's own Q rows.
The 10 bound cases each take one (discount, clip) pair in turn (i mod 4, i mod 5), so every discount and every clip
runs twice on every variant; the all-terminal and no-terminal minibatches come in as host tuples.

The optimizers at their hyperparameters: the update equals oracle.dqn_oracle's, given the device's own gradient, for
every weight and every state plane, on both schedules ("serial": k_optimizer; "branches": k_opt_conv, k_opt_fc1 and
k_opt_small) and at batches and history lengths where those kernels change shape.  Adam's step count t is held at
late steps (0.9^t is subnormal in double at t = 7000) and across every path that trains.  The target's state planes
after update_target_network, and the tensor-core tile images after an Adam or Adadelta step, are pinned as well."""
import random

import numpy as np
import pytest

import kernel_ref as K
import per_oracle as P
from double_oracle import head_restated as double_head
from helpers import make_args
from oracle import dqn_oracle as O
from oracle.replay_oracle import ReplayOracle
from test_gpu_prioritized import _dev, _upload
from test_oracle_flags import BIG, BOUNDS, CLIPS, DISCOUNTS, same

pytestmark = pytest.mark.gpu

F32 = np.float32
ENGINES = ["tcgen05", "fp32"]
SIZE = 400


def _L():
    from simple_dqn_b200 import _lib as L
    return L


def _stream():
    from simple_dqn_b200 import Stream
    return Stream()


def make_net(engine, batch, stream=None, double=False, hist=4, optimizer="rmsprop", seed=3, **flags):
    """Xavier weights with fc1 and fc2 x 3 (Q of order 1), small optimizer state in every plane, a synced target;
    double: the target perturbed so that the two networks prefer different poststate actions."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(4, make_args(batch_size=batch, history_length=hist, random_seed=seed, double_dqn=double,
                                    optimizer=optimizer, **flags), math_mode=engine, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    st = lambda w, scale: (np.abs(rs.randn(*w.shape)) * scale).astype(F32)
    states = {"rmsprop": lambda w: st(w, 1e-4),
              "adam": lambda w: [(rs.randn(*w.shape) * 1e-3).astype(F32), st(w, 1e-5)],
              "adadelta": lambda w: [st(w, 1e-5), st(w, 1e-9), (rs.randn(*w.shape) * 1e-4).astype(F32)]}[optimizer]
    net.set_weights(ws, [states(w) for w in ws])
    net.update_target_network()
    if double:
        net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                        None, which=1)
    return net


_RING = {}


def ring_content(hist=4):
    """A ring of SIZE slots: random frames and actions, rewards drawn from -3..3 and the int64 extremes, 10 %
    terminal."""
    if hist not in _RING:
        ring = ReplayOracle(SIZE, history_length=hist)
        g = np.random.default_rng(17)
        pool = list(range(-3, 4)) + BIG
        for _ in range(SIZE):
            ring.add(int(g.integers(0, 4)), pool[int(g.integers(0, len(pool)))],
                     g.integers(0, 256, (84, 84), dtype=np.uint8), bool(g.random() < 0.1))
        _RING[hist] = ring
    return _RING[hist]


def make_mem(batch, stream, hist=4, **kw):
    from simple_dqn_b200 import ReplayMemory
    ring = ring_content(hist)
    mem = ReplayMemory(SIZE, make_args(batch_size=batch, history_length=hist, **kw), rng="device", stream=stream)
    mem.add_batch(ring.actions, ring.rewards, ring.screens, ring.terminals)
    mem.set_cursor(ring.count, ring.current)
    return ring, mem


def cost_finish(row_costs):
    """k_cost_finish: one fp32 sum in row order, then the division by the row count."""
    tot = F32(0)
    for c in row_costs:
        tot = F32(tot + F32(c))
    return F32(tot / F32(len(row_costs)))


def check_head(net, mb, discount, lo, hi, clip_error, w=None):
    """Deltas, row costs, TD errors (prioritized) and the batch cost of the last step, bit for bit."""
    clip = float(clip_error or 0)
    preq, postq = net.last_q()
    act, rew, term = mb[1], mb[2], mb[4]
    online = net.last_online_postq() if net.double_dqn else None
    if w is not None:
        d, rc, td = P.head_restated(preq, postq, act, rew, term, w, discount, lo, hi, clip, online_postq=online)
        assert same(net.last_td_errors(), td)
    elif online is not None:
        d, rc = double_head(preq, postq, online, act, rew, term, discount, lo, hi, clip)
    else:
        raw, d = K.head_td(preq, postq, act, rew, term, discount, lo, hi, clip)
        rc = (F32(0.5) * raw * raw).sum(axis=1)         # one non-zero delta per row
    assert same(net.last_deltas(), d), np.abs(net.last_deltas() - d).max()
    assert same(net.last_row_costs(), rc)
    assert same(net.last_costs(1)[0], cost_finish(rc)), (net.last_costs(1)[0], cost_finish(rc))


# ------------------------------------------------------------------------------------------------ head and cost
@pytest.mark.parametrize("target", ["vanilla", "double", "prioritized"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("bounds", sorted(BOUNDS))
def test_head_and_cost_at_flag_values(bounds, engine, target):
    i = sorted(BOUNDS).index(bounds)
    discount, clip_error = DISCOUNTS[i % len(DISCOUNTS)], CLIPS[i % len(CLIPS)]
    lo, hi = BOUNDS[bounds]
    stream = _stream()
    per = target == "prioritized"
    ring, mem = make_mem(33, stream, prioritized_replay=per, beta0=0.4)
    if per:                                 # stored priorities spanning 4 decades, every leaf and node rebuilt
        _upload(mem, _L().PTR_PRIORITIES, np.random.default_rng(i).random(SIZE) ** 4 + 1e-3)
        mem.set_cursor(ring.count, ring.current)
    net = make_net(engine, 33, stream, double=target == "double", min_reward=lo, max_reward=hi,
                   discount_rate=discount, clip_error=clip_error)
    mem.seed_device_rng(random.Random(100 + i))
    net.train_fused(mem, 1)
    idx = _dev(mem, _L().PTR_INDEXES, np.int32, 33).astype(np.int64)
    mb = (None, ring.actions[idx], ring.rewards[idx], None, ring.terminals[idx])    # replay_memory.py:76-78
    assert (np.abs(mb[2].astype(np.float64)) > 2.0 ** 53).any()
    w = mem.last_weights if per else None
    if per:
        assert len(np.unique(w)) > 1
    check_head(net, mb, discount, lo, hi, clip_error, w)


@pytest.mark.parametrize("double", [False, True])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("terminals", ["all", "none"])
@pytest.mark.parametrize("bounds", ["half", "inverted", "infinite"])
def test_head_on_all_and_no_terminal_minibatches(bounds, terminals, engine, double):
    lo, hi = BOUNDS[bounds]
    g = np.random.default_rng(len(bounds))
    rew = g.permutation(np.array(list(range(-14, 15)) + BIG, np.int64))
    n = len(rew)
    pre, post = (g.integers(0, 256, (n, 4, 84, 84), dtype=np.uint8) for _ in range(2))
    mb = (pre, g.integers(0, 4, n).astype(np.uint8), rew, post, np.full(n, terminals == "all"))
    net = make_net(engine, n, _stream(), double=double, min_reward=lo, max_reward=hi, discount_rate=0.99,
                   clip_error=1e6)
    net.train(mb, 0)
    check_head(net, mb, 0.99, lo, hi, 1e6)


def test_bounds_past_int32_and_negative_clip_at_construction():
    """Infinite and 3e9 bounds construct and train (the grid above checks what they compute); a negative
    clip_error, which the reference hands Neon's be.clip as crossed bounds, is refused."""
    from simple_dqn_b200 import DeepQNetwork
    g = np.random.default_rng(0)
    states = g.integers(0, 256, (4, 4, 84, 84), dtype=np.uint8)
    mb = (states, np.array([0, 1, 2, 3], np.uint8), np.array([2 ** 31, -(2 ** 31), 2 ** 40, 1], np.int64), states,
          np.array([True, True, False, False]))
    for lo, hi in ((-float("inf"), float("inf")), (-3e9, 3e9), (-3000000000, 3000000000)):
        net = DeepQNetwork(4, make_args(batch_size=4, min_reward=lo, max_reward=hi), math_mode="tcgen05")
        net.train(mb, 0)
        check_head(net, mb, 0.99, lo, hi, 1)
    with pytest.raises(NotImplementedError, match="clip_error"):
        DeepQNetwork(4, make_args(clip_error=-1))


# ------------------------------------------------------------------------------------------------ optimizers
def step_and_check(net, mb, optimizer, t=None, lr=0.00025, decay=0.95):
    """One host-minibatch train step; the weights and every state plane equal the oracle's update of the pre-step
    values with the device's own gradient, bit for bit."""
    w0 = net.get_weights(with_states=False)
    s0 = net.get_states()
    net.train(mb, 0)
    grads = net.get_grads()
    w1, s1 = net.get_weights(with_states=False), net.get_states()
    rows = len(mb[1])
    if optimizer == "rmsprop":
        O.rmsprop_update(w0, [s[0] for s in s0], grads, rows, lr, decay)
    elif optimizer == "adam":
        O.adam_update(w0, s0, grads, rows, t, lr)
    else:
        O.adadelta_update(w0, s0, grads, rows, decay)
    for l in range(5):
        for k in range(net.num_states):
            assert same(s1[l][k], s0[l][k]), (t, l, k)
        assert same(w1[l], w0[l]), (t, l)


def host_minibatch(n, seed, hist=4):
    g = np.random.default_rng(seed)
    return (g.integers(0, 256, (n, hist, 84, 84), dtype=np.uint8), g.integers(0, 4, n).astype(np.uint8),
            g.integers(-3, 4, n).astype(np.int64), g.integers(0, 256, (n, hist, 84, 84), dtype=np.uint8),
            g.random(n) < 0.3)


HYPER = {  # (optimizer, learning_rate, decay_rate)
    "rmsprop": ("rmsprop", 0.00025, 0.95), "rmsprop_lr0.01": ("rmsprop", 0.01, 0.95),
    "rmsprop_lr0": ("rmsprop", 0.0, 0.95), "rmsprop_decay0": ("rmsprop", 0.00025, 0.0),
    "rmsprop_decay0.999": ("rmsprop", 0.00025, 0.999), "adam": ("adam", 0.00025, 0.95),
    "adam_lr0.01": ("adam", 0.01, 0.95), "adadelta": ("adadelta", 0.00025, 0.95),
    "adadelta_decay0.5": ("adadelta", 0.00025, 0.5)}


@pytest.mark.parametrize("sched", ["serial", "branches"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("case", sorted(HYPER))
def test_optimizer_hyperparameters(case, engine, sched):
    opt, lr, decay = HYPER[case]
    net = make_net(engine, 33, _stream() if sched == "branches" else None, optimizer=opt, learning_rate=lr,
                   decay_rate=decay)
    for t in (1, 2):
        step_and_check(net, host_minibatch(33, t), opt, t, lr, decay)


SHAPE_HYPER = {"rmsprop": (0.01, 0.999), "adam": (0.01, 0.95), "adadelta": (0.00025, 0.5)}


@pytest.mark.parametrize("sched", ["serial", "branches"])
@pytest.mark.parametrize("hist", [1, 16])
@pytest.mark.parametrize("batch", [1, 33, 257])
@pytest.mark.parametrize("opt", sorted(SHAPE_HYPER))
def test_optimizer_kernel_shapes(opt, batch, hist, sched):
    """fc2's k_opt_small reduces `rows` per-row partials over 8 lanes (1, 33 and 257 rows: below, above and not a
    multiple of 8); k_opt_conv's conv1 is templated on the history length."""
    lr, decay = SHAPE_HYPER[opt]
    net = make_net("tcgen05", batch, _stream() if sched == "branches" else None, hist=hist, optimizer=opt,
                   learning_rate=lr, decay_rate=decay)
    step_and_check(net, host_minibatch(batch, 3, hist), opt, 1, lr, decay)


@pytest.mark.parametrize("engine,lr", [("tcgen05", 0.00025), ("tcgen05", 0.01), ("fp32", 0.00025)])
def test_adam_late_steps(engine, lr):
    """t = 1, 2, 3, 100, 7000, 20000: the late steps are reached with train_fused at batch 2."""
    stream = _stream()
    _, mem = make_mem(2, stream)
    mem.seed_device_rng(random.Random(5))
    net = make_net(engine, 2, stream, optimizer="adam", learning_rate=lr)
    done = 0
    for t in (1, 2, 3, 100, 7000, 20000):
        if t - 1 > done:
            net.train_fused(mem, t - 1 - done)
        step_and_check(net, host_minibatch(2, t), "adam", t, lr)
        done = t


@pytest.mark.parametrize("engine", ENGINES)
def test_adam_step_count_on_every_path(engine):
    """t counts optimize() calls whichever path ran them."""
    from simple_dqn_b200 import DeviceMinibatch
    stream = _stream()
    ring, mem = make_mem(8, stream, device_minibatch=True)
    mem.seed_device_rng(random.Random(6))
    net = make_net(engine, 8, stream, optimizer="adam")
    check = lambda t: step_and_check(net, host_minibatch(8, t), "adam", t)
    check(1)                                             # host minibatch
    net.train(mem.getMinibatch(), 0)                     # device handle, drawn inside the step (t = 2)
    check(3)
    mem.sample()
    net.train(DeviceMinibatch(mem, sampled=True), 0)     # device handle on a drawn minibatch (t = 4)
    check(5)
    net.train_fused(mem, 4)                              # t = 6..9
    check(10)
    g = np.random.default_rng(0)
    net.step_host(mem, np.zeros(3, np.uint8), np.zeros(3, np.int64), g.integers(0, 256, (3, 84, 84), dtype=np.uint8),
                  np.zeros(3, np.uint8), train_repeat=2)  # t = 11, 12
    check(13)
    net.update_target_network()
    check(14)
    net.set_double_dqn(True)
    check(15)
    net.set_double_dqn(False)
    check(16)
    assert net.train_iterations == 16


@pytest.mark.parametrize("engine", ENGINES)
def test_adam_step_count_across_checkpoints(engine, tmp_path):
    """load_weights into a live net continues its t, as Neon's optimizer object would; a fresh net starts at 1."""
    net = make_net(engine, 8, optimizer="adam")
    for t in (1, 2, 3):
        step_and_check(net, host_minibatch(8, t), "adam", t)
    path = str(tmp_path / "w.pkl")
    net.save_weights(path)
    fresh = make_net(engine, 8, optimizer="adam", seed=9)
    fresh.load_weights(path)
    step_and_check(fresh, host_minibatch(8, 4), "adam", 1)
    net.load_weights(path)
    step_and_check(net, host_minibatch(8, 4), "adam", 4)


@pytest.mark.parametrize("sched", ["serial", "branches"])
@pytest.mark.parametrize("engine", ENGINES)
@pytest.mark.parametrize("opt", ["adam", "adadelta"])
def test_target_sync_copies_every_state_plane(opt, engine, sched):
    net = make_net(engine, 33, _stream() if sched == "branches" else None, optimizer=opt)
    for t in (1, 2):
        net.train(host_minibatch(33, t), 0)
    net.update_target_network()
    for a, b in zip(net.get_weights(which=1, with_states=False), net.get_weights(with_states=False)):
        assert same(a, b)
    for a, b in zip(net.get_states(which=1), net.get_states()):
        assert len(a) == len(b) == O.OPT_STATES[opt]
        for x, y in zip(a, b):
            assert same(x, y)


@pytest.mark.parametrize("sched", ["serial", "branches"])
@pytest.mark.parametrize("batch", [1, 33, 257])
@pytest.mark.parametrize("opt", ["adam", "adadelta"])
def test_tile_images_after_an_update(opt, batch, sched):
    """The hi/lo tile images the optimizer kernels refresh equal a fresh pack of the updated fp32 weights: a twin
    net loaded with those weights predicts the same Q and H1..H4, bit for bit."""
    stream = _stream() if sched == "branches" else None
    net = make_net("tcgen05", batch, stream, optimizer=opt, learning_rate=0.01)
    for t in (1, 2):
        net.train(host_minibatch(batch, t), 0)
    twin = make_net("tcgen05", batch, stream, optimizer=opt, seed=8)
    twin.set_weights(net.get_weights(with_states=False))
    states = host_minibatch(batch, 99)[0]
    assert same(net.predict(states), twin.predict(states))
    for a, b in zip(net.last_activations(), twin.last_activations()):
        assert same(a, b)
