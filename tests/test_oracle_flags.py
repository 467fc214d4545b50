"""The restatements of the TD head (kernel_ref.head_td, double_oracle.head_restated and per_oracle.head_restated at
unit weights) against the reference's own arithmetic, bit for bit, at every value of the flags the head turns into
numbers: --min_reward / --max_reward (type=float, main.py:43-44), --discount_rate and --clip_error.

The reference arithmetic is oracle.dqn_oracle.td_targets (np.clip of the int64 rewards, the target in Python floats
stored as float32), delta = preq - target, the SumSquared row cost before the clip, then the delta clip when
clip_error is truthy (deepqnetwork.py:133-159).  The GPU tests hold the device to the restatements; this file ties
the restatements to the reference, so a restatement that copied a device bug fails here."""
import numpy as np
import pytest

import kernel_ref as K
import per_oracle as P
from double_oracle import head_restated as double_head
from oracle import dqn_oracle as O

F32 = np.float32

# int64 rewards where float64 rounds (2^53 + 1) and at the end of the range
BIG = [2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 63 - 1, -(2 ** 63 - 1)]
BOUNDS = {
    "int_default": (-1, 1),
    "float_default": (-1.0, 1.0),
    "half": (-0.5, 0.5),
    "asymmetric": (-2.5, 3.75),
    "point": (0.25, 0.25),
    "zero": (0, 0),
    "inverted": (1, -1),                # np.clip gives a_max everywhere
    "infinite": (-float("inf"), float("inf")),
    "huge": (-3e9, 3e9),
    "huge_int": (-3000000000, 3000000000),
}
DISCOUNTS = [0.0, 0.5, 0.99, 1.0]
CLIPS = [None, 0, 0.3, 1, 1e6]
TERMINALS = {"mixed": 0.3, "all": 1.1, "none": -0.1}


def same(a, b):
    """Equal bit for bit (so +0 and -0 differ, and inf matches only inf)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def minibatch(terminal_p, num_actions=5, seed=0):
    """Q rows of order 1 and rewards -7..7 plus the int64 extremes, in shuffled order."""
    g = np.random.default_rng(seed)
    rewards = g.permutation(np.array(list(range(-7, 8)) + BIG, np.int64))
    n = len(rewards)
    preq, postq, online = ((g.normal(size=(n, num_actions)) * 2).astype(F32) for _ in range(3))
    actions = g.integers(0, num_actions, n)
    return preq, postq, online, actions, rewards, g.random(n) < terminal_p


def reference(preq, valued_q, actions, rewards, terminals, discount, lo, hi, clip_error):
    """(clipped deltas, row costs, deltas before the clip) by the reference's operations."""
    targets = O.td_targets(preq, valued_q, actions, rewards, terminals, discount, lo, hi)
    deltas = preq - targets
    cost = np.sum(np.square(deltas), axis=1) / F32(2.0)
    raw = deltas.copy()
    if clip_error:
        deltas = np.clip(deltas, -clip_error, clip_error)
    return deltas, cost, raw


@pytest.mark.parametrize("terminals", sorted(TERMINALS))
@pytest.mark.parametrize("bounds", sorted(BOUNDS))
def test_restatements_equal_the_reference(bounds, terminals):
    lo, hi = BOUNDS[bounds]
    preq, postq, online, act, rew, term = minibatch(TERMINALS[terminals])
    n = len(act)
    ones = np.ones(n, F32)
    chosen = postq[np.arange(n), np.argmax(online, axis=1)]     # Double DQN: the online net picks, the target values
    for discount in DISCOUNTS:
        for clip_error in CLIPS:
            clip = float(clip_error or 0)                       # what DeepQNetwork hands the device
            case = (discount, clip_error)
            ref_d, ref_c, ref_raw = reference(preq, postq.max(axis=1), act, rew, term, discount, lo, hi, clip_error)
            raw, d = K.head_td(preq, postq, act, rew, term, discount, lo, hi, clip)
            assert same(d, ref_d) and same(raw, ref_raw), case
            assert same((F32(0.5) * raw * raw).sum(axis=1), ref_c), case     # the row holds one non-zero delta
            d, c, td = P.head_restated(preq, postq, act, rew, term, ones, discount, lo, hi, clip)
            assert same(d, ref_d) and same(c, ref_c), case
            assert same(td, ref_raw[np.arange(n), act]), case

            ref_d, ref_c, ref_raw = reference(preq, chosen, act, rew, term, discount, lo, hi, clip_error)
            d, c = double_head(preq, postq, online, act, rew, term, discount, lo, hi, clip)
            assert same(d, ref_d) and same(c, ref_c), case
            d, c, td = P.head_restated(preq, postq, act, rew, term, ones, discount, lo, hi, clip, online_postq=online)
            assert same(d, ref_d) and same(c, ref_c), case
            assert same(td, ref_raw[np.arange(n), act]), case


def test_the_grid_reaches_what_it_is_for():
    """The cases above are not vacuous: float bounds give fractional targets, crossed bounds give max_reward, the
    extremes survive unbounded clipping (2^53 + 1 rounded to 2^53), and clip_error = 0.3 clips."""
    preq, postq, _, act, rew, term = minibatch(TERMINALS["all"])
    at = lambda t: t[np.arange(len(act)), act]
    for (lo, hi), expect in (((-0.5, 0.5), np.clip(rew, -1, 1) * 0.5),
                             ((1, -1), np.full(len(rew), -1.0)),
                             ((-float("inf"), float("inf")), rew.astype(np.float64))):
        targets = O.td_targets(preq, postq.max(axis=1), act, rew, term, 0.99, lo, hi)
        assert (at(targets) == expect.astype(F32)).all()
    assert F32(2 ** 53 + 1) == F32(2 ** 53) and float(np.int64(2 ** 53 + 1)) == 2.0 ** 53
    raw, d = K.head_td(preq, postq, act, rew, term, clip=0.3)
    assert (np.abs(at(d)) == F32(0.3)).any() and (np.abs(at(raw)) > F32(0.3)).any()
