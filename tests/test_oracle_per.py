"""The prioritized-replay oracle (tests/per_oracle.py) on the CPU: its drawable set against the reference-pinned
acceptance test, its tree descent against a brute-force draw, its weights, its random-stream consumption, and its
weighted train step against the vanilla oracle and torch autograd."""
import random

import numpy as np
import pytest
import torch
from scipy import stats

import per_oracle as P
from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle
from test_oracle_dqn import torch_forward


def _ring(size, hist, count, current, terminal_p, seed):
    r = ReplayOracle(size, 2, 2, history_length=hist, batch_size=8)
    g = np.random.default_rng(seed)
    r.terminals[:] = g.random(size) < terminal_p
    r.count, r.current = count, current
    return r


RINGS = [  # (size, count, current): unwrapped, full and wrapped, write pointer at both ends
    (200, 120, 120), (200, 200, 0), (200, 200, 57), (200, 200, 199), (300, 300, 290), (64, 40, 40)]


@pytest.mark.parametrize("hist", [1, 4, 16])
@pytest.mark.parametrize("terminal_p", [0.0, 0.05, 0.4])
def test_leaf_mask_is_the_reference_acceptance_test(hist, terminal_p):
    for k, (size, count, current) in enumerate(RINGS):
        r = _ring(size, hist, count, current, terminal_p, seed=k)
        mask = P.valid_mask(r.terminals, r.count, r.current, hist)
        for i in range(size):
            ref = hist <= i <= count - 1 and r.accept(i)
            assert mask[i] == ref, (size, count, current, i)


@pytest.mark.parametrize("hist", [1, 4, 16])
def test_draws_never_return_an_invalid_slot(hist):
    g = np.random.default_rng(hist)
    for k, (size, count, current) in enumerate(RINGS):
        r = _ring(size, hist, count, current, 0.3, seed=10 + k)
        mask = P.valid_mask(r.terminals, r.count, r.current, hist)
        if not mask.any():
            continue
        prio = g.random(size) ** 3          # spans orders of magnitude
        sums, mins = P.build(np.where(mask, prio, 0.0))
        rng = MT19937.from_python(random.Random(k))
        for _ in range(5):
            idx, w = P.draw(sums, mins, rng, 40, count)
            assert mask[idx].all()
            assert (w > 0).all() and (w <= 1).all()


def test_layout_at_one_million_slots():
    n, off = P.layout(1 << 20)
    assert n == [1 << 20, 1 << 15, 1 << 10, 32, 1]          # four levels under the root
    assert off[-1] * 8 < 8.3 * 2 ** 20
    n, off = P.layout(50)
    assert n == [50, 2, 1] and off == [0, 64, 96, 128]


@pytest.mark.parametrize("size", [50, 1000, 40000])
def test_descent_equals_brute_force_on_dyadic_priorities(size):
    """Integer priorities: every partial sum is exact, so the descent is the textbook cumsum / searchsorted draw."""
    g = np.random.default_rng(size)
    leaves = g.integers(0, 9, size).astype(np.float64)
    sums, _ = P.build(leaves)
    cum = np.cumsum(leaves)
    assert sums[-1][0] == cum[-1]
    for mass in np.concatenate([g.random(500) * cum[-1], [0.0, cum[-1] - 0.5]]):
        ref = int(np.searchsorted(cum, mass, side="right"))
        slot, leaf = P.descend(sums, float(mass))
        assert slot == ref and leaf == leaves[ref]


def test_rounding_fallback_never_returns_a_zero_leaf():
    leaves = np.zeros(100)
    leaves[[3, 40, 77]] = [0.1, 0.2, 0.3]
    sums, _ = P.build(leaves)
    slot, leaf = P.descend(sums, float(sums[-1][0]) * 1.5)    # a mass beyond the total: last positive child
    assert slot == 77 and leaf == 0.3


def test_alpha_zero_is_stratified_uniform_with_unit_weights():
    r = _ring(500, 4, 500, 123, 0.05, seed=3)
    per = P.PEROracle(r, alpha=0.0, beta0=0.4, beta_steps=10)
    per.update(np.arange(4, 200), np.linspace(-3, 3, 196))       # alpha = 0: every priority stays 1
    assert (per.prio == 1.0).all()
    valid = np.nonzero(per.leaves() > 0)[0]
    rng = MT19937.from_python(random.Random(9))
    check = MT19937.from_python(random.Random(9))
    for step in range(3):
        idx, w = per.draw(rng, 32)
        assert (w == np.float32(1.0)).all()
        seg = len(valid) / 32
        for i in range(32):
            mass = P.random_from_words(check.genrand_uint32(), check.genrand_uint32()) * seg + i * seg
            assert idx[i] == valid[int(np.floor(mass))]


def test_draw_frequencies_match_priorities():
    r = _ring(96, 4, 96, 50, 0.05, seed=4)
    mask = P.valid_mask(r.terminals, r.count, r.current, 4)
    g = np.random.default_rng(5)
    leaves = np.where(mask, g.random(96) * 4 + 0.05, 0.0)
    sums, mins = P.build(leaves)
    rng = MT19937.from_python(random.Random(5))
    counts = np.zeros(96)
    for _ in range(1500):
        idx, _ = P.draw(sums, mins, rng, 32, 96)
        np.add.at(counts, idx, 1)
    assert counts[~mask].sum() == 0
    exp = leaves[mask] / leaves.sum() * counts.sum()
    assert stats.chisquare(counts[mask], exp).pvalue > 1e-3


@pytest.mark.parametrize("batch", [1, 8, 32, 400])
def test_one_draw_consumes_two_words_per_sample(batch):
    host = random.Random(11)
    for _ in range(300):
        host.random()                      # start mid-key so that the draw crosses a regeneration
    rng = MT19937.from_python(host)
    r = _ring(1000, 4, 1000, 10, 0.02, seed=6)
    per = P.PEROracle(r)
    expect = [host.random() for _ in range(batch)]
    idx, _ = per.draw(rng, batch)
    assert rng.words_drawn == 2 * batch
    assert rng.state625() == list(host.getstate()[1])
    # and random.random() is the word pair the draw uses
    rng2 = MT19937.from_python(random.Random(11))
    h2 = random.Random(11)
    for _ in range(50):
        assert P.random_from_words(rng2.genrand_uint32(), rng2.genrand_uint32()) == h2.random()


def test_beta_anneals_and_weights_follow_baselines():
    assert P.beta_at(0, 0.4, 100) == 0.4
    assert P.beta_at(50, 0.4, 100) == 0.4 + 0.6 * 0.5
    assert P.beta_at(500, 0.4, 100) == 1.0
    # baselines: max_weight = (p_min N)^-beta, weight = (p N)^-beta / max_weight; the rarest slot weighs 1
    assert P.weight(0.5, 2.0, 0.5, 10.0, 0.7) == np.float32(1.0)
    assert P.weight(1.5, 2.0, 0.5, 10.0, 0.0) == np.float32(1.0)
    np.testing.assert_allclose(P.weight(1.5, 2.0, 0.5, 10.0, 1.0), 1 / 3, rtol=1e-7)


def test_update_last_occurrence_wins_and_max_priority():
    r = _ring(100, 4, 100, 0, 0.0, seed=7)
    per = P.PEROracle(r, alpha=0.5, eps=1e-6)
    per.update([10, 20, 10], [4.0, -0.25, 0.01])
    assert per.prio[10] == (0.01 + 1e-6) ** 0.5
    assert per.prio[20] == (0.25 + 1e-6) ** 0.5
    assert per.max_priority == 4.0 + 1e-6
    cur = r.current
    per.add(0, 0, np.zeros((2, 2), np.uint8), False)
    assert per.prio[cur] == (4.0 + 1e-6) ** 0.5 and r.current == cur + 1


def _batch(n, a, seed, terminal_p=0.3):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (n, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (n, 4, 84, 84)).astype(np.uint8)
    return (pre, rs.randint(0, a, n).astype(np.uint8), rs.randint(-3, 4, n).astype(np.int64), post,
            rs.rand(n) < terminal_p)


def test_unit_weights_equal_the_vanilla_step_bit_for_bit():
    ws = O.xavier_init(4, seed=2)
    a = O.DQNOracle(4, batch_size=8, weights=ws)
    b = O.DQNOracle(4, batch_size=8, weights=ws)
    for i in range(3):
        mb = _batch(8, 4, 20 + i)
        ca = a.train(mb)
        cb = P.train_weighted(b, mb, np.ones(8, np.float32))
        assert ca == cb
        assert (a.last["deltas"] == b.last["deltas"]).all()
        for x, y in zip(a.weights + a.states, b.weights + b.states):
            assert (x == y).all()


def test_weighted_gradient_matches_torch_autograd_of_weighted_huber():
    ws = O.xavier_init(6, seed=4)
    for w in (ws[3], ws[4]):
        w *= np.float32(3)
    mb = _batch(16, 6, 3)
    wts = np.random.default_rng(1).uniform(0.1, 1.0, 16).astype(np.float32)
    net = O.DQNOracle(6, batch_size=16, weights=ws)
    P.train_weighted(net, mb, wts)
    pre, act, rew, post, term = mb
    with torch.no_grad():
        maxpost = torch_forward([torch.tensor(w) for w in ws], torch.tensor(post)).max(dim=1).values.numpy()
    tw = [torch.tensor(w, requires_grad=True) for w in ws]
    preq = torch_forward(tw, torch.tensor(pre))
    r = np.clip(rew, -1, 1).astype(np.float64)
    y = torch.tensor(np.where(term, r, r + 0.99 * maxpost.astype(np.float64)).astype(np.float32))
    d = preq[torch.arange(16), torch.tensor(act.astype(np.int64))] - y
    loss = (torch.tensor(wts) * torch.nn.functional.huber_loss(d, torch.zeros_like(d), reduction="none",
                                                               delta=1.0)).sum()
    loss.backward()
    assert (np.abs(d.detach().numpy()) > 1).any() and (np.abs(d.detach().numpy()) < 1).any()   # both huber branches
    for g, t in zip(net.last["grads"], tw):
        ref = t.grad.numpy()
        assert np.linalg.norm(g - ref) <= 1e-4 * np.linalg.norm(ref)
    np.testing.assert_allclose(net.last["td"], d.detach().numpy(), rtol=1e-5, atol=1e-6)


def test_head_restated_with_unit_weights_is_the_vanilla_head():
    from double_oracle import head_restated as vanilla_double
    g = np.random.default_rng(8)
    preq, postq, onl = (g.normal(size=(32, 6)).astype(np.float32) for _ in range(3))
    act = g.integers(0, 6, 32)
    rew = g.integers(-3, 4, 32)
    term = g.random(32) < 0.3
    d1, c1 = vanilla_double(preq, postq, onl, act, rew, term)
    d2, c2, _ = P.head_restated(preq, postq, act, rew, term, np.ones(32, np.float32), online_postq=onl)
    assert (d1 == d2).all() and (c1 == c2).all()
