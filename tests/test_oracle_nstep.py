"""The n-step restatement (tests/nstep_oracle.py) against independent statements of the same rules: at N = 1 the
reference's replay oracle and kernel_ref.head_td bit for bit, CPython's own random.randint filtered by a window test
written from its definition, exact rational arithmetic for the return, and torch autograd for the gradient."""
import random
from fractions import Fraction

import numpy as np
import pytest

import kernel_ref as K
import nstep_oracle as NS
from oracle.mt19937 import MT19937
from oracle.replay_oracle import ReplayOracle, synthetic_ring
from test_oracle_flags import BOUNDS, DISCOUNTS, minibatch, same

F32 = np.float32


def _ring(size, hist, count=None, current=None, seed=0, terminal_p=0.05, batch=32):
    ring = ReplayOracle(size, screen_height=2, screen_width=3, history_length=hist, batch_size=batch)
    synthetic_ring(ring, seed=seed, terminal_p=terminal_p, count=count, current=current)
    return ring


def blocked_by_definition(index, hist, n, current):
    """The window index-H .. index+N-1 is cut by the write pointer when one of its consecutive slot pairs (j, j+1) is
    the pair (current - 1, current): slot current holds the oldest frame, slot current - 1 the newest."""
    return any(j + 1 == current for j in range(index - hist, index + n - 1))


# ---------------------------------------------------------------------------------------------- N = 1 is the reference
@pytest.mark.parametrize("hist", [1, 4, 16])
@pytest.mark.parametrize("wrapped", [False, True])
def test_draw_at_one_step_is_the_reference(hist, wrapped):
    ring = _ring(600, hist, count=None if wrapped else 400, current=117 if wrapped else 400, seed=hist)
    for i in range(ring.size):
        assert NS.accept(ring, i, 1) == ring.accept(i)
    for seed in range(5):
        a, b = MT19937.from_python(random.Random(seed)), MT19937.from_python(random.Random(seed))
        idx, words = NS.sample_indexes(ring, a, 1)
        assert (idx == ring.sample_indexes(b)).all()
        assert words == b.words_drawn and a.state625() == b.state625()
    mask = NS.valid_mask(ring.terminals, ring.count, ring.current, hist, 1)
    ref = np.array([hist <= i <= ring.count - 1 and ring.accept(i) for i in range(ring.size)])
    assert (mask == ref).all()


def test_gather_at_one_step_is_the_reference():
    ring = _ring(300, 4, current=50, seed=3)
    idx = np.array([4, 49, 54, 120, 299])
    pre, act, rew, post, term = NS.gather(ring, idx, 1)
    rpre, ract, rrew, rpost, rterm = ring.gather(idx)
    assert (pre == rpre[:5]).all() and (post == rpost[:5]).all() and (act == ract).all()
    assert (rew[:, 0] == rrew).all() and (term[:, 0] == rterm).all()


@pytest.mark.parametrize("bounds", sorted(BOUNDS))
@pytest.mark.parametrize("double", [False, True])
def test_head_at_one_step_is_kernel_ref(bounds, double):
    lo, hi = BOUNDS[bounds]
    preq, postq, online, act, rew, term = minibatch(0.3, seed=5)
    n = len(act)
    for discount in DISCOUNTS:
        for clip in (0.0, 0.3, 1.0):
            if double:
                chosen = postq[np.arange(n), np.argmax(online, axis=1)]
                vq = np.repeat(chosen[:, None], postq.shape[1], axis=1)   # every column the Double DQN choice
                raw, d = K.head_td(preq, vq, act, rew, term, discount, lo, hi, clip)
                nd, nc, ntd = NS.head_restated(preq, postq, act, rew, term, discount, lo, hi, clip, online_postq=online)
            else:
                raw, d = K.head_td(preq, postq, act, rew, term, discount, lo, hi, clip)
                nd, nc, ntd = NS.head_restated(preq, postq, act, rew, term, discount, lo, hi, clip)
            assert same(nd, d) and same(ntd, raw[np.arange(n), act])
            assert same(nc, (F32(0.5) * raw * raw).sum(axis=1))


# ---------------------------------------------------------------------------------------------- the draw
@pytest.mark.parametrize("hist", [1, 4, 16])
@pytest.mark.parametrize("n", [1, 2, 3, 5, 16])
@pytest.mark.parametrize("wrapped", [False, True])
def test_draw_equals_cpython_randint_and_the_window_definition(hist, n, wrapped):
    """Every index, the words consumed and the generator state equal CPython's random.randint(H, count - N) filtered
    by the definition of the window test and the :65 terminal test."""
    size = 400
    for current in ([0, 1, hist, hist + 1, 150, 399] if wrapped else [200]):
        ring = _ring(size, hist, count=None if wrapped else 200, current=current, seed=n * 31 + hist)
        for i in range(hist, ring.count - n + 1):
            assert NS.crosses_write_pointer(i, hist, n, current) == blocked_by_definition(i, hist, n, current)
        py = random.Random(current + 7 * n)
        mt = MT19937.from_python(py)
        idx, words = NS.sample_indexes(ring, mt, n, batch=40)
        expect, trials = [], 0
        while len(expect) < 40:
            i = py.randint(hist, ring.count - n)
            trials += 1
            if not blocked_by_definition(i, hist, n, current) and not ring.terminals[i - hist:i].any():
                expect.append(i)
        assert list(idx) == expect
        assert mt.state625() == list(py.getstate()[1])   # the same words consumed
        assert words >= trials                            # randbelow's retries take words without making a trial


def test_window_edges_of_the_write_pointer():
    """current at index - H and index + N is drawable, at index - H + 1 and index + N - 1 it is not."""
    for hist in (1, 4, 16):
        for n in (1, 2, 3, 16):
            i = 100
            assert not NS.crosses_write_pointer(i, hist, n, i - hist)
            assert NS.crosses_write_pointer(i, hist, n, i - hist + 1)
            assert NS.crosses_write_pointer(i, hist, n, i + n - 1)
            assert not NS.crosses_write_pointer(i, hist, n, i + n)


def test_valid_mask_is_accept():
    for hist, n, count, current in ((4, 3, 300, 300), (1, 16, 400, 37), (16, 5, 400, 0), (4, 1, 400, 399)):
        ring = _ring(400, hist, count=count, current=current, seed=hist + n, terminal_p=0.1)
        mask = NS.valid_mask(ring.terminals, count, current, hist, n)
        ref = [hist <= i <= count - n and NS.accept(ring, i, n) for i in range(400)]
        assert (mask == np.array(ref)).all()


# ---------------------------------------------------------------------------------------------- the return
REWARDS = list(range(-7, 8)) + [2 ** 53 + 1, -(2 ** 53 + 1), 2 ** 63 - 1, -(2 ** 63 - 1)]


@pytest.mark.parametrize("bounds", sorted(BOUNDS))
@pytest.mark.parametrize("n", [1, 2, 3, 5, 16])
def test_return_within_its_rounding_bound_of_exact_arithmetic(bounds, n):
    lo, hi = BOUNDS[bounds]
    g = np.random.default_rng(n)
    for discount in DISCOUNTS:
        for cut in list(range(n)) + [None]:        # a terminal at every position of the window, and none
            rew = g.choice(np.array(REWARDS, dtype=object), n)
            term = [k == cut for k in range(n)]
            R, gk, t = NS.n_step_return(rew, term, discount, lo, hi)
            assert t == (cut is not None)
            m = n if cut is None else cut + 1
            c = [Fraction(NS.clip_reward(r, lo, hi)) for r in rew[:m]]
            gam = Fraction(discount)
            exact = sum(gam ** k * c[k] for k in range(m))
            scale = sum(abs(gam ** k * c[k]) for k in range(m))
            assert abs(Fraction(R) - exact) <= 2 * n * Fraction(1, 2 ** 53) * scale, (discount, cut)
            if cut is None:
                assert abs(Fraction(gk) - gam ** n) <= n * Fraction(1, 2 ** 53) * gam ** n * 2


def test_return_truncation_and_gamma_powers_are_exact_on_dyadic_rewards():
    """With gamma = 0.5 and small integer rewards every operation is exact: R and g are the textbook values."""
    rew = [1, -1, 1, 1, -1]
    for cut in range(5):
        term = [k == cut for k in range(5)]
        R, g, t = NS.n_step_return(rew, term, 0.5)
        assert t and R == sum(0.5 ** k * rew[k] for k in range(cut + 1)) and g == 0.5 ** cut
    R, g, t = NS.n_step_return(rew, [False] * 5, 0.5)
    assert not t and g == 0.5 ** 5 and R == sum(0.5 ** k * rew[k] for k in range(5))
    assert NS.target(rew, [False] * 5, 2.0, 0.5) == R + 0.5 ** 5 * 2.0
    assert NS.target(rew, [False, True, False, False, False], 2.0, 0.5) == 0.5


# ---------------------------------------------------------------------------------------------- the gradient
@pytest.mark.parametrize("n", [2, 3, 16])
@pytest.mark.parametrize("clip", [0.3, 1.0])
def test_head_gradient_is_autograd_of_the_huber_loss(n, clip):
    torch = pytest.importorskip("torch")
    g = np.random.default_rng(n)
    b, A = 33, 5
    preq = (g.normal(size=(b, A)) * 2).astype(F32)
    postq = (g.normal(size=(b, A)) * 2).astype(F32)
    act = g.integers(0, A, b)
    rew = g.integers(-3, 4, (b, n))
    term = g.random((b, n)) < 0.15
    d, cost, td = NS.head_restated(preq, postq, act, rew, term, 0.99, -1, 1, clip)
    y = torch.tensor([NS.target(rew[i], term[i], postq[i].max(), 0.99) for i in range(b)], dtype=torch.float64)
    q = torch.tensor(preq.astype(np.float64), requires_grad=True)
    qa = q[torch.arange(b), torch.tensor(act)]
    loss = torch.nn.functional.huber_loss(qa, y, reduction="sum", delta=clip)
    loss.backward()
    np.testing.assert_allclose(d, q.grad.numpy(), rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(cost, 0.5 * (qa.detach().numpy() - y.numpy()) ** 2, rtol=1e-5, atol=1e-6)
