"""Bootstrapped DQN heads on the device against tests/bootstrap_oracle.py, each stage fed the device's own inputs so that
errors do not carry over.  No stage uses expf or logf, so everything is bit for bit: the masks at the read-back ring
slots, theta of all three slots, the per-head targets and deltas, the row costs, TD errors and cost, dtheta, dZ4 and its
fp16 planes, fc2's gradient and its update under every optimizer, the mean-over-heads Q rows and predict at every
active head; on both engines and both schedules, with Double DQN, prioritized replay, n-step returns, random shift and
target_steps = 0.  Also the masks of a ring slot across steps, fused runs against single steps, ring steps against
host-tuple steps at p = 1, head switches between replays of a captured predict graph, the agent loop with the documented
binding (a head per training episode, the mean in evaluation), the launched kernels against REM's, checkpoints, the
target sync and the refusals."""
import os
import random

import numpy as np
import pytest

import bootstrap_oracle as BOOT
from helpers import make_args
from test_gpu_distributional import ENGINES, _L, _gather, _optimize, _ring_pair, _same_state, _slot_h4, _state

pytestmark = pytest.mark.gpu

F32 = np.float32


def _bnet(mode, A=4, K=10, p=0.5, clip=1.0, batch=32, hist=4, stream=None, double=False, seed=3, scale=3.0,
          optimizer="rmsprop", target_steps=10000, discount=0.99, shift=0):
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(A, make_args(batch_size=batch, history_length=hist, random_seed=seed, double_dqn=double,
                                    bootstrapped=True, bootstrap_heads=K, bootstrap_p=p, clip_error=clip,
                                    optimizer=optimizer, target_steps=target_steps, discount_rate=discount,
                                    random_shift=shift), math_mode=mode, stream=stream)
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


def _check_train_step(net, before, slots, actions, rewards, terminals, post, clip, discount=0.99, w=None,
                      separate=True, nstep=False):
    """Every stage of the last train step, bit for bit, fed the device's own inputs.  before = (weights, states) ahead
    of the step, slots the ring slots it read (the mask's key); rewards / terminals are (batch, N) windows; post the
    poststates the target slots read (None: not checked, the states were shifted); separate: the target network is not
    the online one."""
    A, K, b = net.num_actions, net.num_heads, len(actions)
    m = net.last_bootstrap_masks()
    assert (m == BOOT.masks(net.bootstrap_seed, slots, K, net.bootstrap_p)).all()
    theta = net.last_heads()
    two = net.double_dqn and separate
    h4 = net.last_activations()[3]
    w5 = before[0][4]
    assert (theta[0].reshape(b, A * K) == BOOT.logits(h4, w5.T)).all()
    tws = net.get_weights(which=1, with_states=False) if separate else before[0]
    if post is not None:
        assert (theta[1].reshape(b, A * K) == BOOT.logits(_slot_h4(net, tws, post), tws[4].T)).all()
        if two:
            assert (theta[2].reshape(b, A * K) == BOOT.logits(_slot_h4(net, before[0], post), w5.T)).all()
    rewards, terminals = np.asarray(rewards), np.asarray(terminals)
    returns = [BOOT.n_step_return(rewards[i], terminals[i], discount) for i in range(b)]
    q, T, D, cost, err, g = BOOT.head(theta, actions, returns, m, clip, double=two, nstep=nstep, w=w)
    preq, postq = net.last_q()
    assert (preq == q[0]).all() and (postq == q[1]).all()
    if two:
        assert (net.last_online_postq() == q[2]).all()
    assert (net.last_head_targets() == T).all()
    assert (net.last_head_deltas() == D).all()
    rc = net.last_row_costs()
    assert (rc == cost).all()
    if w is not None:
        assert (net.last_td_errors() == err).all()
    tot = F32(0)
    for c in rc:
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(b))
    assert (net.last_head_grads() == g).all()
    dz4 = net.last_dz()[3]
    for i in range(b):
        assert (dz4[i] == BOOT.dz4(h4[i], w5.T, actions[i], g[i])).all(), i
    if net.math_mode == "tcgen05":
        hi16, lo16 = net.last_dz4_planes()
        ehi, elo = BOOT.fp16_planes(dz4)
        assert (hi16.view(np.uint16) == ehi.view(np.uint16)).all() and (lo16.view(np.uint16) == elo.view(np.uint16)).all()
    grad = BOOT.fc2_grad(h4, g, actions, A)
    assert (net.get_grads()[4] == grad).all()
    w_new, s_new = _optimize(net.optimizer, w5, before[1][4], grad, b)
    ws, ss = _state(net)
    assert (ws[4] == w_new).all()
    for k in range(net.num_states):
        assert (ss[4][k] == s_new[k]).all(), k
    return m, g


def _ring_slots(mem, batch):
    from test_gpu_prioritized import _dev
    return _dev(mem, _L().PTR_INDEXES, np.int32, batch).astype(np.int64)


# ---------------------------------------------------------------------------------------------------- predict
PREDICT = [  # (mode, batch, A, K)
    ("tcgen05", 1, 1, 1), ("fp32", 64, 32, 200), ("tcgen05", 65, 18, 10), ("fp32", 33, 4, 2),
]


@pytest.mark.parametrize("mode,batch,A,K", PREDICT)
def test_predict_at_every_head(mode, batch, A, K):
    """theta equals the restated fp32 dot products; predict at h = -1 (the default) is the mean over the heads, and at
    every h >= 0 theta's column h; the Xavier draw is the REM layout's."""
    from oracle import dqn_oracle as O
    from simple_dqn_b200 import DeepQNetwork
    fresh = DeepQNetwork(A, make_args(batch_size=batch, random_seed=5, bootstrapped=True, bootstrap_heads=K),
                         math_mode=mode)
    for x, y in zip(fresh.get_weights(with_states=False), O.xavier_init(A * K, 5)):
        assert (x == y).all()
    net = _bnet(mode, A=A, K=K, batch=batch)
    assert net.active_head == -1
    ws = net.get_weights(with_states=False)
    assert ws[4].shape == (A * K, 512)
    states = np.random.RandomState(batch + A).randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    q = net.predict(states)
    h4 = net.last_activations()[3]
    theta = net.last_heads()[0]
    assert (theta.reshape(batch, A * K) == BOOT.logits(h4, ws[4].T)).all()
    assert (q == BOOT.predict_q(theta)).all()
    for h in range(K):
        net.set_active_head(h)
        assert (net.predict(states) == theta[..., h]).all(), h
    assert net.active_head == K - 1
    net.set_active_head(-1)
    assert (net.predict(states) == q).all()


# ---------------------------------------------------------------------------------------------------- train step
STEP = [  # (batch, A, K, p, n, clip, double, per, hist, discount, shift)
    (32, 4, 10, 0.5, 1, 1.0, False, False, 4, 0.99, 0), (1, 1, 1, 0.9, 3, 0.0, True, True, 4, 1.0, 0),
    (65, 18, 200, 0.5, 1, 1.0, True, False, 4, 0.99, 0), (64, 32, 2, 0.1, 3, 0.0, False, True, 4, 0.99, 0),
    (33, 4, 10, 1.0, 3, 1.0, True, True, 1, 0.99, 4), (257, 4, 10, 0.5, 1, 0.0, False, False, 4, 0.0, 0),
]


@pytest.mark.parametrize("mode,sched", ENGINES)
@pytest.mark.parametrize("batch,A,K,p,n,clip,double,per,hist,discount,shift", STEP)
def test_train_step_stages(mode, sched, batch, A, K, p, n, clip, double, per, hist, discount, shift):
    from simple_dqn_b200 import DeviceMinibatch, Stream
    from test_gpu_prioritized import _upload
    stream = Stream() if sched == "branches" else None
    ring, mem = _ring_pair(batch=batch, hist=hist, stream=stream, prioritized_replay=per, beta0=0.4, terminal_p=0.1)
    ring.actions[:] = np.random.RandomState(batch).randint(0, A, len(ring.actions))
    _upload(mem, _L().PTR_ACTIONS, ring.actions)
    mem.set_n_step(n)
    net = _bnet(mode, A=A, K=K, p=p, clip=clip, batch=batch, hist=hist, stream=stream, double=double,
                discount=discount, shift=shift)
    for step in range(2):
        before = _state(net)
        idx = np.array(random.Random(batch * 7 + n + step).sample(range(hist, 3000 - n + 1), batch), np.int32)
        mem.set_indexes(idx)
        net.train(DeviceMinibatch(mem, sampled=True))
        slots = _ring_slots(mem, batch)
        mb = _gather(ring, slots, n)
        m, _ = _check_train_step(net, before, slots, mb[1].astype(np.int64), mb[2], mb[4], None if shift else mb[3],
                                 clip, discount=discount, w=mem.last_weights if per else None, nstep=n > 1)
    if p == 1.0:
        assert (m == 1).all()
    elif batch * K >= 64:
        assert 0 < m.mean() < 1


@pytest.mark.parametrize("optimizer", ["rmsprop", "adam", "adadelta"])
@pytest.mark.parametrize("target_steps", [10000, 0])
def test_optimizers_and_target_steps_zero(optimizer, target_steps):
    """A host-minibatch step at p = 1 under every optimizer (Adam's step scalar comes from the new head), with and
    without a separate target network, Double DQN on; the engine alternates."""
    from helpers import random_minibatch
    mode = "tcgen05" if (optimizer == "adam") == (target_steps == 0) else "fp32"
    clip = 0.0 if optimizer == "adadelta" else 1.0
    net = _bnet(mode, A=4, K=10, p=1.0, clip=clip, batch=33, optimizer=optimizer, target_steps=target_steps,
                double=True)
    before = _state(net)
    pre, act, rew, post, term = random_minibatch(33, 4, 5)
    net.train((pre, act, rew, post, term))
    _check_train_step(net, before, np.arange(33), act.astype(np.int64), rew[:, None], term[:, None], post, clip,
                      separate=target_steps != 0)


# ---------------------------------------------------------------------------------------------------- masks on the ring
@pytest.mark.parametrize("mode,sched", ENGINES)
def test_fused_run_equals_single_steps(mode, sched):
    """train_fused(3) equals three train_fused(1) calls (replays of the captured step graph) of a twin on an identically
    seeded ring, bit for bit, and every replay's masks are the stated ones of the slots it drew."""
    from simple_dqn_b200 import Stream
    nets = []
    for single in (False, True):
        stream = Stream() if sched == "branches" else None
        _, mem = _ring_pair(stream=stream)
        net = _bnet(mode, K=10, p=0.5, stream=stream)
        random.seed(5)
        mem.seed_device_rng(random)
        if single:
            for _ in range(3):
                net.train_fused(mem, 1)
                assert (net.last_bootstrap_masks() == BOOT.masks(net.bootstrap_seed, _ring_slots(mem, 32), 10,
                                                                  0.5)).all()
        else:
            net.train_fused(mem, 3)
        nets.append(net)
    assert (nets[0].last_costs(3) == nets[1].last_costs(3)).all()
    assert (nets[0].last_bootstrap_masks() == nets[1].last_bootstrap_masks()).all()
    _same_state(nets[0], nets[1])


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_masks_belong_to_the_ring_slot_and_host_tuples(mode):
    """A ring slot drawn in two steps carries the same mask; at p = 1 two ring steps equal the same steps from host
    tuples bit for bit; at p < 1 a host tuple is refused before any device work, and a materialised DeviceMinibatch
    still trains from the ring."""
    from simple_dqn_b200 import DeviceMinibatch, Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream)
    net = _bnet(mode, K=10, p=0.5, stream=stream)
    idx = np.array(random.Random(1).sample(range(50, 2900), 32), np.int32)
    masks = []
    for step in range(2):
        mem.set_indexes(np.roll(idx, step))
        net.train(DeviceMinibatch(mem, sampled=True))
        masks.append(net.last_bootstrap_masks())
    assert (np.roll(masks[0], 1, axis=0) == masks[1]).all()
    assert 0 < masks[0].mean() < 1
    mb = _gather(ring, idx, 1)
    before = _state(net)
    with pytest.raises(NotImplementedError, match="bootstrap"):
        net.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
    ws, _ = _state(net)
    for x, y in zip(ws, before[0]):
        assert (x == y).all()
    mem.set_indexes(idx)
    dm = DeviceMinibatch(mem, sampled=True)
    np.asarray(dm[0])   # materialise it
    net.train(dm)
    assert (net.last_bootstrap_masks() == masks[0]).all()

    one = _bnet(mode, K=10, p=1.0, stream=stream)
    twin = _bnet(mode, K=10, p=1.0, stream=Stream())
    for step in range(2):
        idx = np.array(random.Random(step).sample(range(50, 2900), 32), np.int32)
        mem.set_indexes(idx)
        one.train(DeviceMinibatch(mem, sampled=True))
        mb = _gather(ring, idx, 1)
        twin.train((mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]))
        assert (one.last_costs(1) == twin.last_costs(1)).all()
        assert (one.last_head_grads() == twin.last_head_grads()).all()
        assert (one.last_bootstrap_masks() == 1).all() and (twin.last_bootstrap_masks() == 1).all()
        _same_state(one, twin)


# ---------------------------------------------------------------------------------------------------- acting
@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_head_switch_between_replays_of_the_captured_predict(mode):
    """The fast-path predict graph is captured once; switching the head between its replays changes the Q it returns
    to the new head's column, and the host predict and predict_device agree at every head."""
    import ctypes as C
    from simple_dqn_b200 import StateBuffer, Stream
    stream = Stream()
    net = _bnet(mode, K=10, stream=stream)
    sb = StateBuffer(make_args(), stream=stream)
    rs = np.random.RandomState(1)
    for _ in range(4):
        sb.add(rs.randint(0, 256, (84, 84)).astype(np.uint8))
    ds = sb.getStateMinibatch()
    mean = net.predict(ds)
    theta = net.last_heads()[0][0]
    assert (mean[0] == BOOT.predict_q(theta)).all() and (mean[1:] == 0).all()
    L = _L()
    for h in (3, 0, 9, -1, 7):
        net.set_active_head(h)
        fast = net.predict(ds)
        want = BOOT.predict_q(theta, h)
        assert (fast[0] == want).all() and (fast[1:] == 0).all(), h
        host = net.predict(np.asarray(ds))
        assert (host[0] == want).all(), h
        qp = net.device_view(L.NET_PTR_Q_ONLINE, (32, 4)).ptr
        L.call("b200dqn_net_predict_device", net._h, C.c_void_p(ds.device_ptr()), 1, C.c_void_p(qp), net._stream)
        assert (net._read_f32(L.NET_PTR_Q_ONLINE, (32, 4))[0] == want).all(), h


class _BootAgent:
    """src/agent.py's _restartRandom, step, train and test, restated (eps = 0 throughout, no replay), with the lines
    INTEGRATION.md adds for bootstrapped heads marked (+).  Every greedy predict is logged with the head the binding
    says it must act on."""

    def __init__(self, env, net, buf, history_length=4, random_starts=8):
        self.env, self.net, self.buf = env, net, buf
        self.history_length, self.random_starts = history_length, random_starts
        self.head = None          # what the binding says is active
        self.heads, self.log, self.terminals = [], [], {"train": 0, "test": 0}
        self.phase = None

    def _restartRandom(self):                                 # agent.py:29-39
        self.env.restart()
        for _ in range(random.randint(self.history_length, self.random_starts) + 1):
            self.env.act(0)
            if self.env.isTerminal():
                self.env.restart()
            self.buf.add(self.env.getScreen())

    def step(self):                                           # agent.py:48-85 at exploration rate 0
        q = self.net.predict(self.buf.getStateMinibatch())
        self.log.append((self.phase, self.head, self.net.active_head, q[0].copy(), self.net.last_heads()[0][0].copy()))
        reward = self.env.act(int(np.argmax(q[0])))
        screen = self.env.getScreen()
        terminal = self.env.isTerminal()
        self.buf.add(screen)
        if terminal:
            self.terminals[self.phase] += 1
            self._restartRandom()
        return terminal

    def _sample(self):
        self.head = self.net.sample_head()
        self.heads.append(self.head)

    def train(self, steps):                                   # agent.py:96-116 (no replay, no updates here)
        self.phase = "train"
        self._sample()                                        # (+) the episode test left running gets a fresh head
        for _ in range(steps):
            if self.step():
                self._sample()                                # (+) step restarted the game: a new training episode

    def test(self, steps):                                    # agent.py:118-124
        self.phase = "test"
        self.net.set_active_head(-1)                          # (+) evaluation acts on the mean over the heads
        self.head = -1
        self._restartRandom()
        for _ in range(steps):
            self.step()


def test_agent_binding_samples_heads_in_training_and_evaluates_on_the_mean():
    """The reference's agent loop with INTEGRATION.md's binding, train / test / train on the synthetic environment:
    every training predict acts on the head drawn at the start of train() or at the last training terminal, every test
    predict on the mean over the heads, including after test's own _restartRandom and its terminals; the heads are the
    net's own RandomState draws."""
    from simple_dqn_b200 import StateBuffer, Stream
    from simple_dqn_b200.synthetic_env import SyntheticEnvironment
    stream = Stream()
    net = _bnet("tcgen05", K=10, stream=stream)
    random.seed(3)
    agent = _BootAgent(SyntheticEnvironment(4, seed=2, episode_mean=8), net, StateBuffer(make_args(), stream=stream))
    agent._restartRandom()
    agent.train(40)
    agent.test(30)
    agent.train(40)
    assert agent.terminals["train"] >= 2 and agent.terminals["test"] >= 1, agent.terminals
    for phase, want, active, q, theta in agent.log:
        assert active == want, (phase, want, active)
        assert (q == BOOT.predict_q(theta, want)).all(), (phase, want)
    assert {w for p, w, _, _, _ in agent.log if p == "test"} == {-1}
    assert len(set(agent.heads)) >= 2
    rs = np.random.RandomState(net.bootstrap_seed % (1 << 32))
    assert agent.heads == [int(rs.randint(10)) for _ in agent.heads]


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_launches_are_rem_minus_the_mixture_draw(mode):
    """The kernels a fused step actually launches, by label from the in-graph timeline: a bootstrapped step launches
    REM's kernels with head_boot for head_rem and without rem_alpha.  launches_per_step, counted at the launch sites
    while the step was captured, is REM's minus one, and so is the static count it gives before the first fused step
    (which the library keeps as it was for every other head)."""
    from collections import Counter
    from simple_dqn_b200 import Stream
    from test_gpu_rem import _rnet
    L = _L()
    stream = Stream()
    _, mem = _ring_pair(stream=stream)
    random.seed(1)
    mem.seed_device_rng(random)
    labels, counts, static = {}, {}, {}
    for head in ("rem", "boot"):
        n = _rnet(mode, stream=stream) if head == "rem" else _bnet(mode, stream=stream)
        static[head] = n.launches_per_step()
        n.train_fused(mem, 1)
        counts[head] = n.launches_per_step()
        L.ktrace_begin(0)
        n.train_fused(mem, 1)      # recaptured with one timeline slot per launch
        stream.synchronize()
        labels[head] = Counter(r[0] for r in L.ktrace_end())
    assert counts["boot"] == counts["rem"] - 1, counts
    assert static["boot"] == static["rem"] - 1, static
    assert labels["rem"]["rem_alpha"] == 1 and labels["rem"]["head_rem"] == 1
    want = labels["rem"] - Counter({"rem_alpha": 1, "head_rem": 1}) + Counter({"head_boot": 1})
    assert labels["boot"] == want, (labels["boot"], labels["rem"])


# ---------------------------------------------------------------------------------------------------- state
def test_checkpoints_target_sync_and_refusals(tmp_path):
    """Both checkpoint layouts round-trip; a REM checkpoint with as many heads loads; the target sync copies fc2; the
    refusals."""
    from helpers import random_minibatch
    from simple_dqn_b200 import DeepQNetwork
    from test_gpu_rem import _rnet
    net = _bnet("tcgen05", optimizer="adam", p=1.0)
    net.train(random_minibatch(32, 4, 3))
    for layout in ("neon-1.3.0", "pre-1.0"):
        path = os.path.join(str(tmp_path), "boot_%s.pkl" % layout)
        net.save_weights(path, layout=layout)
        other = _bnet("fp32", optimizer="adam", seed=9)
        other.load_weights(path)
        _same_state(net, other)
        scalar = DeepQNetwork(4, make_args(), math_mode="tcgen05")
        with pytest.raises(AssertionError):
            scalar.load_weights(path)
    rem = _rnet("tcgen05", K=10, optimizer="adam")
    rpath = os.path.join(str(tmp_path), "rem.pkl")
    rem.save_weights(rpath)
    net.load_weights(rpath)
    assert (net.get_weights(with_states=False)[4] == rem.get_weights(with_states=False)[4]).all()
    net.update_target_network()
    assert (net.get_weights(which=1, with_states=False)[4] == net.get_weights(with_states=False)[4]).all()
    L = _L()
    for k in range(net.num_states):
        a, b = np.empty((4 * 10, 512), F32), np.empty((4 * 10, 512), F32)
        L.call("b200dqn_net_get_state", net._h, 0, 4, k, L.np_ptr(a), None)
        L.call("b200dqn_net_get_state", net._h, 1, 4, k, L.np_ptr(b), None)
        assert (a == b).all()
    for kw in ({"bootstrap_heads": 0}, {"bootstrap_heads": 201}, {"bootstrap_p": 0.0}, {"bootstrap_p": 2.0},
               {"rem": True, "num_heads": 10}, {"quantile_regression": True, "num_quantiles": 10}):
        args = dict(bootstrapped=True, bootstrap_heads=10)
        args.update(kw)
        with pytest.raises(AssertionError):
            DeepQNetwork(4, make_args(**args), math_mode="tcgen05")
    for kw in ({"dueling": True}, {"munchausen": True}):
        with pytest.raises(NotImplementedError, match="bootstrap"):
            DeepQNetwork(4, make_args(bootstrapped=True, **kw), math_mode="tcgen05")
    with pytest.raises(NotImplementedError, match="bootstrap"):
        net.comm_init(bytes(128), 0, 2)
    for h in (-2, 10):
        with pytest.raises(AssertionError):
            net.set_active_head(h)
    with pytest.raises(AssertionError):
        rem.set_active_head(0)
    with pytest.raises(AssertionError):
        net.last_deltas()
    for sel in (L.NET_PTR_REM_ALPHAS, L.NET_PTR_REM_COUNTER, L.NET_PTR_QUANTILES, L.NET_PTR_IQN_TAU_COUNTER):
        with pytest.raises(AssertionError):
            net._read_f32(sel, (1,))
    with pytest.raises(AssertionError):
        rem.last_head_targets()


@pytest.mark.parametrize("mode", ["tcgen05", "fp32"])
def test_fused_trajectory_against_a_numpy_bootstrapped_step(mode):
    """Five fused steps against tests/bootstrap_oracle.numpy_step (oracle.dqn_oracle's forward, backward and RMSProp
    with this head) on the same minibatches and masks: cost within 1e-3, every layer's update within rel-L2 2e-2."""
    from helpers import rel_l2
    from simple_dqn_b200 import Stream
    stream = Stream()
    ring, mem = _ring_pair(stream=stream, terminal_p=0.05)
    net = _bnet(mode, K=200, p=0.5, stream=stream)
    ws, ss = _state(net)
    ows, oss = [w.copy() for w in ws], [s[0].copy() for s in ss]
    tws = net.get_weights(which=1, with_states=False)
    w0 = [w.copy() for w in ws]
    random.seed(9)
    mem.seed_device_rng(random)
    for step in range(5):
        net.train_fused(mem, 1)
        idx = _ring_slots(mem, 32)
        mb = _gather(ring, idx, 1)
        m = BOOT.masks(net.bootstrap_seed, idx, 200, 0.5)
        assert (net.last_bootstrap_masks() == m).all()
        ref, _, _ = BOOT.numpy_step(ows, oss, tws, (mb[0], mb[1], mb[2][:, 0], mb[3], mb[4][:, 0]), 200, m)
        cost = float(net.last_costs(1)[0])
        assert abs(cost - ref) <= 1e-3 * abs(ref), (cost, ref)
    got = net.get_weights(with_states=False)
    for l in range(5):
        assert rel_l2(got[l] - w0[l], ows[l] - w0[l]) <= 2e-2, l
