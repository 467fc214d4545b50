"""The uniform index draw of getMinibatch (replay_memory.py:55-69; csrc/replay.cuh sample_block) at its edges, bit for
bit against CPython's own ``random.randint`` filtered by ReplayOracle's acceptance test: every accepted index in
acceptance order, the words consumed, and the MT19937 state after every draw (the host ``random`` with rng="python",
the device stream with rng="device").

The edges are those of sample_block: a batch around the sampler's 256 threads, a draw width n = count - H at and
around powers of two (where n.bit_length() changes), a draw that starts at MT19937 position 0, 623 or 624 (key
regeneration before the first word, after it, or at once), H = 1 and 16, the write pointer at both ends of the ring,
unwrapped and wrapped rings, and rings with no terminals, many terminals or a single drawable index.

Sampler-only cases use 4x4 screens, so even a 1M-slot ring is 16 MB.  Every ring is checked to have a drawable index
and fewer than 1e5 expected words per draw before the device draws from it: the uniform sampler retries until it has
a full minibatch."""
import random

import numpy as np
import pytest

from helpers import make_args
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring

pytestmark = pytest.mark.gpu


class _CountingRandom(random.Random):
    """CPython's generator, counting 32-bit output words: randint draws through getrandbits(k <= 32), one word each."""
    words = 0

    def getrandbits(self, k):
        self.words += 1
        return super().getrandbits(k)


def accept_mask(terminals, count, current, hist):
    """ReplayOracle.accept for every index in [0, count) (False below hist, where randint never lands)."""
    t = np.concatenate([[0], np.cumsum(np.asarray(terminals[:count], np.int64))])
    idx = np.arange(count)
    ok = idx >= hist
    ok &= ~((idx >= current) & (idx - hist < current))               # :61, the write pointer
    ok &= t[idx] == t[np.maximum(idx - hist, 0)]                     # :65, no terminal among the hist frames before
    return ok


def check_mask_against_oracle(mask, terminals, count, current, hist, size, probe=3000):
    orc = ReplayOracle(8, screen_height=4, screen_width=4, history_length=hist)   # a shell over the test's arrays
    orc.size, orc.count, orc.current, orc.terminals = size, count, current, np.asarray(terminals, np.bool_)
    n = count - hist
    if n <= probe:
        probes = np.arange(hist, count)
    else:
        probes = np.unique(np.concatenate([np.arange(hist, hist + 64), np.arange(count - 64, count),
                                           np.arange(max(hist, current - 40), min(count, current + 40)),
                                           np.random.default_rng(count).integers(hist, count, probe)]))
    assert [bool(mask[i]) for i in probes] == [orc.accept(int(i)) for i in probes]


def guard_drawable(mask, hist, count, batch):
    """Never hand the device a ring it would spin on: a drawable index, and a bounded expected draw length."""
    drawable = int(mask.sum())
    n = count - hist
    assert drawable > 0, "no drawable index"
    words = batch * (1 << n.bit_length()) / drawable
    assert words < 1e5, "expected %.0f words per draw" % words
    return drawable


def expected_draw(rnd, mask, hist, count, batch):
    """replay_memory.py:55-69 with CPython's randint: accepted indexes in acceptance order, and the words consumed."""
    w0 = rnd.words
    out = []
    while len(out) < batch:
        index = rnd.randint(hist, count - 1)
        if mask[index]:
            out.append(index)
    return np.array(out, np.int64), rnd.words - w0


def set_python_random(seed, pos):
    """Seed the process-global `random`, then move its MT19937 position to `pos` (0: a freshly regenerated key)."""
    key = random.Random(seed).getstate()[1][:624]
    random.setstate((3, tuple(key) + (pos,), None))


def make_ring(size, count, current, hist, batch, terminals, rng, stream=None):
    from simple_dqn_b200 import ReplayMemory
    mem = ReplayMemory(size, make_args(screen_height=4, screen_width=4, history_length=hist, batch_size=batch),
                       rng=rng, stream=stream)
    g = np.random.default_rng(size + hist)
    mem.add_batch(g.integers(0, 4, size, dtype=np.uint8), g.integers(-1, 2, size, dtype=np.int64),
                  g.integers(0, 256, (size, 4, 4), dtype=np.uint8), terminals)
    mem.set_cursor(count, current)
    return mem


def terminals_with(size, p, seed):
    if p == 0:
        return np.zeros(size, np.uint8)
    return (np.random.default_rng(seed).random(size) < p).astype(np.uint8)


def run_draws(mem, terminals, count, current, hist, batch, rng_mode, draws, seed, pos):
    size = mem.size
    mask = accept_mask(terminals, count, current, hist)
    check_mask_against_oracle(mask, terminals, count, current, hist, size)
    guard_drawable(mask, hist, count, batch)
    set_python_random(seed, pos)
    host_before = random.getstate()
    rnd = _CountingRandom()
    rnd.setstate(host_before)
    mask_list = mask.tolist()
    for d in range(draws):
        idx, words = expected_draw(rnd, mask_list, hist, count, batch)
        mem.getMinibatch()
        assert (mem.last_indexes == idx).all(), d
        assert mem.last_words_consumed == words, (d, mem.last_words_consumed, words)
        if rng_mode == "python":
            assert random.getstate()[1] == rnd.getstate()[1], d
        else:
            assert tuple(int(x) for x in mem.read_device_rng()) == rnd.getstate()[1], d
    if rng_mode == "device":
        assert random.getstate() == host_before                 # the device stream never touches the host's
    return rnd.words


# (size, count, current, hist, batch, terminal p or "one", MT position at the first draw, rng mode)
_B = 5000
CASES = {
    # batch around the sampler's 256 threads and far above it (H = 4, n = 4996, wrapped)
    "batch1": (_B, _B, 1234, 4, 1, 0.0, 623, "python"),
    "batch2": (_B, _B, 1234, 4, 2, 0.3, 0, "device"),
    "batch255": (_B, _B, 1234, 4, 255, 0.3, 624, "python"),
    "batch256": (_B, _B, 1234, 4, 256, 0.0, 623, "device"),
    "batch257": (_B, _B, 1234, 4, 257, 0.3, 0, "python"),
    "batch1000": (_B, _B, 1234, 4, 1000, 0.3, 624, "device"),
    "batch4096": (_B, _B, 1234, 4, 4096, 0.3, 623, "python"),
    # history lengths, with the write pointer at 0, 1, H - 1, H, H + 1 and count - 1
    "h1_cur0": (3000, 3000, 0, 1, 257, 0.05, 624, "python"),
    "h1_curlast": (3000, 2000, 1999, 1, 257, 0.3, 623, "device"),
    "h2_cur1": (3000, 3000, 1, 2, 257, 0.3, 623, "device"),
    "h4_curhm1": (3000, 2500, 3, 4, 257, 0.05, 0, "python"),
    "h4_curh": (3000, 3000, 4, 4, 300, 0.3, 624, "device"),
    "h4_curhp1": (3000, 2600, 5, 4, 256, 0.0, 623, "python"),
    "h16_curh": (3000, 3000, 16, 16, 257, 0.05, 623, "device"),
    "h16_curhp1": (3000, 2000, 17, 16, 255, 0.05, 0, "python"),
    "h16_curhm1": (3000, 3000, 15, 16, 1000, 0.0, 624, "python"),
    # draw widths n = count - H at and around powers of two
    "n1": (8, 5, 5, 4, 257, 0.0, 623, "python"),
    "n1_wrapped": (17, 17, 0, 16, 256, 0.0, 624, "device"),
    "n2": (64, 6, 6, 4, 256, 0.0, 0, "device"),
    "n3_one_drawable": (16, 7, 7, 4, 257, "one", 623, "python"),
    "n255_wrapped": (259, 259, 1, 4, 257, 0.3, 624, "device"),
    "n256": (600, 257, 0, 1, 1000, 0.0, 0, "python"),
    "n256_wrapped": (260, 260, 259, 4, 257, 0.05, 623, "device"),
    "n257_wrapped": (261, 261, 260, 4, 4096, 0.3, 623, "device"),
    "n65536": (70000, 65540, 65540, 4, 256, 0.3, 624, "python"),
    "n65536_wrapped": (65538, 65538, 2, 2, 4096, 0.0, 0, "device"),
    "n65537_wrapped": (65541, 65541, 0, 4, 1000, 0.05, 623, "python"),
    "n65537_h16": (70000, 65553, 65553, 16, 257, 0.05, 0, "device"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_uniform_draw_at_its_edges(case):
    size, count, current, hist, batch, p, pos, rng = CASES[case]
    if p == "one":                     # n = 3: indexes 4, 5, 6; a terminal in slot 4 leaves index 4 alone drawable
        terminals = np.zeros(size, np.uint8)
        terminals[4] = 1
    else:
        terminals = terminals_with(size, p, seed=size + batch)
    mem = make_ring(size, count, current, hist, batch, terminals, rng)
    if p == "one":
        assert accept_mask(terminals, count, current, hist).sum() == 1
    draws = 12 if batch <= 2 else 4
    run_draws(mem, terminals, count, current, hist, batch, rng, draws, seed=len(case) * 1009 + batch, pos=pos)


_BIG = 1_048_600


@pytest.mark.parametrize("n,current,batch,rng,pos", [((1 << 20) - 1, 1048578, 4096, "python", 623),
                                                     ((1 << 19) + 1, 3, 1000, "device", 0)])
def test_uniform_draw_on_a_1m_ring(n, current, batch, rng, pos):
    """n = 2^20 - 1 (every 20-bit word in range) and 2^19 + 1 (about half out of range), the ring unwrapped."""
    hist = 4
    count = n + hist
    terminals = terminals_with(_BIG, 0.05, seed=n)
    mem = make_ring(_BIG, count, current, hist, batch, terminals, rng)
    run_draws(mem, terminals, count, current, hist, batch, rng, 4, seed=n, pos=pos)


def test_long_run_of_key_regenerations():
    """Batch 4096, 300 consecutive draws on a 70k-slot ring: thousands of key regenerations, each draw compared."""
    size, hist, batch = 70000, 4, 4096
    terminals = terminals_with(size, 0.05, seed=70)
    current = 31337
    mem = make_ring(size, size, current, hist, batch, terminals, "python")
    mask = accept_mask(terminals, size, current, hist)
    # the numpy mask restates ReplayOracle.sample_indexes: the two agree on a prefix of the stream
    set_python_random(404, 624)
    orc = ReplayOracle(8, screen_height=4, screen_width=4, history_length=hist, batch_size=batch)
    orc.size, orc.count, orc.current, orc.terminals = size, size, current, terminals.astype(np.bool_)
    rng = MT19937.from_python(random)
    rnd = _CountingRandom()
    rnd.setstate(random.getstate())
    for _ in range(2):
        assert (orc.sample_indexes(rng, batch_size=512) == expected_draw(rnd, mask.tolist(), hist, size, 512)[0]).all()
    assert rnd.getstate()[1] == tuple(rng.state625())
    words = run_draws(mem, terminals, size, current, hist, batch, "python", 300, seed=405, pos=0)
    assert words > 2000 * 624                                    # at least 2000 key regenerations were compared


# ---------------------------------------------------------------------------------------------- inside the step
def _indexes(mem):
    from simple_dqn_b200 import _lib as L
    view = mem.device_view(L.PTR_INDEXES, np.int32, (mem.batch_size,))
    return L.download(mem.device, view.ptr, (mem.batch_size,), np.int32, mem._stream)


@pytest.mark.parametrize("path", ["train_fused", "step_host"])
@pytest.mark.parametrize("hist", [1, 16])
@pytest.mark.parametrize("batch", [1, 257, 512])
def test_draws_inside_the_fused_step(path, hist, batch):
    """The draw captured at the head of the step graph equals the oracle's, step by step.  step_host appends frames
    before each step and keeps the host `random` in lock-step, including after somebody else drew from it."""
    from simple_dqn_b200 import DeepQNetwork, ReplayMemory, Stream
    st = Stream()
    orc = ReplayOracle(3000, history_length=hist, batch_size=batch)
    synthetic_ring(orc, seed=hist + batch, block=150, terminal_p=0.05)
    mem = ReplayMemory(3000, make_args(history_length=hist, batch_size=batch),
                       rng="device" if path == "train_fused" else "python", stream=st)
    mem.add_batch(orc.actions, orc.rewards, orc.screens, orc.terminals)
    mem.set_cursor(orc.count, orc.current)
    net = DeepQNetwork(4, make_args(history_length=hist, batch_size=batch), math_mode="tcgen05", stream=st)
    set_python_random(batch * 7 + hist, 623 if batch == 257 else 624)
    rng = MT19937.from_python(random)
    g = np.random.default_rng(batch)
    for step in range(3):
        guard_drawable(accept_mask(orc.terminals, orc.count, orc.current, hist), hist, orc.count, batch)
        if path == "train_fused":
            net.train_fused(mem, 1)
            idx = orc.sample_indexes(rng)
            assert (_indexes(mem) == idx).all(), step
            net.last_costs(1)
            assert [int(x) for x in mem.read_device_rng()] == rng.state625(), step
        else:
            k = 2 + step
            a, r = g.integers(0, 4, k, dtype=np.uint8), g.integers(-1, 2, k, dtype=np.int64)
            s, t = g.integers(0, 256, (k, 84, 84), dtype=np.uint8), g.random(k) < 0.05
            for i in range(k):
                orc.add(a[i], r[i], s[i], t[i])
            if step == 1:
                random.random()                                  # somebody else draws: the state goes up again
            rng = MT19937.from_python(random)
            net.step_host(mem, a, r, s, t, train_repeat=1)
            idx = orc.sample_indexes(rng)
            assert (_indexes(mem) == idx).all(), step
            assert mem.last_words_consumed == rng.words_drawn, step
            assert list(random.getstate()[1]) == rng.state625(), step
