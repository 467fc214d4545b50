"""The ring half of the fused train step: which ring a cached step graph reads, the frame gather on a full 1M-slot
ring whose upper windows lie past 2^32 bytes, and k_gather / getState at every frame size.  Every reference is exact:
ReplayOracle, a numpy restatement of the ring's content, or the host-minibatch path of the same build."""
import gc
import random

import numpy as np
import pytest

from helpers import make_args
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, decode_frame_tag, synthetic_ring
from test_gpu_sampler import accept_mask, guard_drawable

pytestmark = pytest.mark.gpu

F32 = np.float32


def _net(mode, batch=32, hist=4, stream=None, double=False, seed=3):
    """Trained-looking online weights, non-zero RMSProp state, and a target network that differs from the online one."""
    from simple_dqn_b200 import DeepQNetwork
    net = DeepQNetwork(4, make_args(batch_size=batch, history_length=hist, random_seed=seed, double_dqn=double),
                       math_mode=mode, stream=stream)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for w in ws])
    net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                    None, which=1)
    return net


def _net_state(net):
    return net.get_weights(with_states=False), net.get_states(), net.get_weights(which=1, with_states=False)


def _assert_same_state(a, b):
    for x, y in zip(a[0] + a[2], b[0] + b[2]):
        assert (x == y).all()
    for x, y in zip(a[1], b[1]):
        for p, q in zip(x, y):
            assert (p == q).all()


def _indexes(mem):
    from simple_dqn_b200 import _lib as L
    view = mem.device_view(L.PTR_INDEXES, np.int32, (mem.batch_size,))
    return L.download(mem.device, view.ptr, (mem.batch_size,), np.int32, mem._stream)


# ------------------------------------------------------------------------------------------------ ring identity
def _small_ring(size, seed, current, rng, stream, device_minibatch=False, **kw):
    from simple_dqn_b200 import ReplayMemory
    orc = ReplayOracle(size)
    synthetic_ring(orc, seed=seed, block=50, terminal_p=0.01, current=current)
    mem = ReplayMemory(size, make_args(**kw), rng=rng, device_minibatch=device_minibatch, stream=stream)
    mem.add_batch(orc.actions, orc.rewards, orc.screens, orc.terminals)
    mem.set_cursor(orc.count, orc.current)
    return mem


def _frames(step):
    g = np.random.default_rng(100 + step)
    return (g.integers(0, 4, 2, dtype=np.uint8), g.integers(-1, 2, 2, dtype=np.int64),
            g.integers(0, 256, (2, 84, 84), dtype=np.uint8), g.random(2) < 0.1)


def _one_step(net, mem, path, step):
    from simple_dqn_b200 import DeviceMinibatch
    if path == "train_fused":
        net.train_fused(mem, 1)
    elif path == "train":                               # a device minibatch: the draw rides in the step graph
        net.train(mem.getMinibatch(), 0)
    elif path == "train_sampled":                       # drawn first: the step graph without the sampler
        mem.sample()
        net.train(DeviceMinibatch(mem, sampled=True), 0)
    else:
        net.step_host(mem, *_frames(step), train_repeat=1)


_RNG = {"train_fused": "device", "train": "python", "train_sampled": "device", "step_host": "python"}
IDENTITY = ([(p, m, False) for p in ("train_fused", "train", "train_sampled", "step_host") for m in ("tcgen05", "fp32")]
            + [("train_fused", "tcgen05", True)])


@pytest.mark.parametrize("path,mode,per", IDENTITY)
def test_step_graphs_follow_the_ring_they_were_captured_on(path, mode, per):
    """A net captures its step graph on ring A; A is destroyed and ring B, which may get A's address, takes its place.
    Three steps on B through the same path equal, bit for bit, the same steps of a twin net that never saw A."""
    from simple_dqn_b200 import Stream
    st = Stream()
    rng, dm = _RNG[path], path == "train"
    net = _net(mode, stream=st)
    mem_a = _small_ring(600, seed=1, current=77, rng=rng, stream=st, device_minibatch=dm)
    random.seed(10)
    _one_step(net, mem_a, path, 0)
    net.last_costs(1)
    after_a = _net_state(net)
    handle_a = mem_a._h.value
    del mem_a
    gc.collect()

    def ring_b():
        return _small_ring(5000, seed=2, current=1234, rng=rng, stream=st, device_minibatch=dm,
                           prioritized_replay=per, beta_steps=10)

    tries = []
    for _ in range(6):                                  # look for a ring that got A's address
        tries.append(ring_b())
        if tries[-1]._h.value == handle_a:
            break
    mem_b = tries.pop()
    reused = mem_b._h.value == handle_a
    del tries
    gc.collect()
    print("ring handle reused:", reused)

    twin = _net(mode, stream=st, seed=5)
    twin.set_weights(after_a[0], after_a[1])
    twin.set_weights(after_a[2], None, which=1)
    twin_b = ring_b()
    runs = []
    for n, mem in ((net, mem_b), (twin, twin_b)):
        random.seed(20)
        for step in range(1, 4):
            _one_step(n, mem, path, step)
        costs = n.last_costs(3)
        runs.append((costs, _net_state(n), mem.read_device_rng(), random.getstate(),
                     mem.priorities if per else None))
    (ca, sa, ra, ha, pa), (cb, sb, rb, hb, pb) = runs
    assert (ca == cb).all(), (ca, cb)
    _assert_same_state(sa, sb)
    assert (ra == rb).all()
    assert ha == hb
    if per:
        assert (pa == pb).all()


# ---------------------------------------------------------------------------------------------- the 1M-slot ring
BIG, BLK = 1_000_000, 10_000
PAST_4G = 608_702     # the whole window of an index from here up lies past 2^32 bytes of 84x84 frames


class BigRing:
    """A full 1M-slot 84x84 ring of distinct frames: a 10k random block tiled through it, each frame's first four
    bytes overwritten with its slot number, so that a window read from anywhere else differs."""

    def __init__(self, hist, batch, stream=None):
        from simple_dqn_b200 import ReplayMemory
        g = np.random.default_rng(1000 + hist)
        self.hist, self.batch, self.current = hist, batch, 123_457
        self.base = g.integers(0, 256, (BLK, 84, 84), dtype=np.uint8)
        self.actions = g.integers(0, 4, BIG, dtype=np.uint8)
        self.rewards = g.integers(-1, 2, BIG, dtype=np.int64)
        self.terminals = g.random(BIG) < 0.005
        self.mem = ReplayMemory(BIG, make_args(history_length=hist, batch_size=batch), rng="device", stream=stream)
        for s in range(0, BIG, BLK):
            self.mem.add_batch(self.actions[s:s + BLK], self.rewards[s:s + BLK], self.frames(np.arange(s, s + BLK)),
                               self.terminals[s:s + BLK])
        self.mem.set_cursor(BIG, self.current)
        guard_drawable(accept_mask(self.terminals, BIG, self.current, hist), hist, BIG, batch)

    def frames(self, slots):
        f = self.base[slots % BLK]
        tags = slots.astype(np.uint32)[..., None].view(np.uint8)
        f.reshape(slots.shape + (-1,))[..., :4] = tags
        return f

    def oracle(self):
        orc = ReplayOracle(8, history_length=self.hist, batch_size=self.batch)   # a shell over the arrays above
        orc.size, orc.count, orc.current, orc.terminals = BIG, BIG, self.current, self.terminals
        return orc

    def check_minibatch(self, mb, idx):
        pre, a, r, post, t = (np.asarray(x) for x in mb)
        slots = idx[:, None] - self.hist + np.arange(self.hist)
        assert (decode_frame_tag(pre) == slots).all() and (decode_frame_tag(post) == slots + 1).all()
        assert (pre == self.frames(slots)).all() and (post == self.frames(slots + 1)).all()
        assert (a == self.actions[idx]).all() and (r == self.rewards[idx]).all() and (t == self.terminals[idx]).all()


def fused_equals_host(ring, mode, double=False, per=False):
    """3 steps of train_fused (in two calls) against the host-minibatch path (getMinibatch through k_gather, then
    train), or against sample + train_sampled on a prioritized ring.  Returns the indexes drawn."""
    from simple_dqn_b200 import DeviceMinibatch
    mem, stream = ring.mem, ring.mem._stream_obj
    out, drawn = [], []
    for fused in (True, False):
        net = _net(mode, batch=ring.batch, hist=ring.hist, stream=stream, double=double)
        if per:                     # beta0 = 1: the weights do not depend on the ring's running sampling count
            mem.set_prioritized(True, beta0=1.0)
        random.seed(77)
        rng = MT19937.from_python(random)
        mem.seed_device_rng(random)
        if fused:
            net.train_fused(mem, 1)
            net.train_fused(mem, 2)
            idx = _indexes(mem)
        else:
            orc = ring.oracle()
            for _ in range(3):
                if per:
                    mem.sample()
                    net.train(DeviceMinibatch(mem, sampled=True), 0)
                    continue
                mb = mem.getMinibatch()
                idx = orc.sample_indexes(rng)
                assert (mem.last_indexes == idx).all()
                ring.check_minibatch(mb, idx)
                drawn.append(idx)
                net.train(mb, 0)
            idx = _indexes(mem)
        costs = net.last_costs(3)
        out.append((costs, _net_state(net), mem.read_device_rng(), idx, mem.priorities if per else None))
        del net
    if per:
        mem.set_prioritized(False)
    else:
        assert [int(x) for x in out[1][2]] == rng.state625()
    (ca, sa, ra, ia, pa), (cb, sb, rb, ib, pb) = out
    assert (ca == cb).all(), (ca, cb)
    _assert_same_state(sa, sb)
    assert (ra == rb).all() and (ia == ib).all()
    if per:
        assert (pa == pb).all()
    return np.concatenate(drawn) if drawn else ia


@pytest.fixture(scope="module")
def big_ring():
    from simple_dqn_b200 import Stream
    ring = BigRing(4, 32, stream=Stream())
    yield ring
    ring.mem = None
    gc.collect()


FUSED_1M = ["tcgen05", "tcgen05_b257", "tcgen05_h16", "fp32", "double", "prioritized"]


@pytest.mark.parametrize("case", FUSED_1M)
def test_fused_gather_on_a_full_1m_ring(big_ring, case):
    """The conv1 frame gather reads windows in place, up to 7 GB into the ring; k_gather copies them out.  At most
    two 7 GB rings are alive at once: the shared H = 4 ring and a case's own."""
    from simple_dqn_b200 import Stream
    ring = big_ring
    if case == "tcgen05_b257":
        ring = BigRing(4, 257, stream=Stream())
    elif case == "tcgen05_h16":
        ring = BigRing(16, 32, stream=Stream())
    mode = "fp32" if case == "fp32" else "tcgen05"
    idx = fused_equals_host(ring, mode, double=case == "double", per=case == "prioritized")
    assert (idx >= PAST_4G).any(), idx
    del ring
    gc.collect()


# ------------------------------------------------------------------------------------------- every frame size
FRAME_SIZES = [(5, 7), (4, 4), (84, 84), (210, 160), (480, 480), (512, 512)]


@pytest.mark.parametrize("hw", FRAME_SIZES, ids=["%dx%d" % hw for hw in FRAME_SIZES])
@pytest.mark.parametrize("hist", [1, 4, 16])
def test_gather_and_get_state_at_every_frame_size(hw, hist):
    """k_gather takes its bulk-copy path for frames that are a multiple of 16 B and fit in a block's shared memory
    (4x4 ... 480x480), else its byte loop (5x7, 512x512).  Minibatch bytes and scalars, and getState(i) for every i in
    [-count, count), equal ReplayOracle's."""
    from simple_dqn_b200 import ReplayMemory
    h, w = hw
    size, batch = 48, 8
    orc = ReplayOracle(size, screen_height=h, screen_width=w, history_length=hist, batch_size=batch)
    synthetic_ring(orc, seed=h * w + hist, terminal_p=0.02, current=13)
    guard_drawable(accept_mask(orc.terminals, orc.count, orc.current, hist), hist, orc.count, batch)
    mem = ReplayMemory(size, make_args(screen_height=h, screen_width=w, history_length=hist, batch_size=batch),
                       rng="python")
    mem.add_batch(orc.actions, orc.rewards, orc.screens, orc.terminals)
    mem.set_cursor(orc.count, orc.current)
    random.seed(h + w + hist)
    rng = MT19937.from_python(random)
    for _ in range(2):
        got = mem.getMinibatch()
        idx = orc.sample_indexes(rng)
        ref = orc.gather(idx)
        assert (mem.last_indexes == idx).all()
        for a, b in zip(got, ref):
            assert a.shape == b.shape and (np.asarray(a) == np.asarray(b)).all()
    for i in range(-orc.count, orc.count):
        assert (mem.getState(i) == orc.getState(i)).all(), i
