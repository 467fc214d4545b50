"""tests/head_oracle.py against independent computations (CPU): both rules within fp32 rounding bounds of float64 at
every action count and row count the GPU sweep runs, the butterfly against a lane-by-lane scalar simulation, and the
orders the rules fix shown to be observable (a sequential row sum and a reversed warp order differ from them), so that a
bit-for-bit comparison on the device tells them apart."""
import numpy as np
import pytest

import head_oracle as H

F32 = np.float32
U = 2.0 ** -24


def _gamma(n):
    return n * U / (1 - n * U)


def _h4(rows, seed):
    """Rectified activations of order 1 with about half of them zero, as fc1's output."""
    g = np.random.default_rng(seed)
    return np.maximum(g.standard_normal((rows, H.HIDDEN)), 0).astype(F32)


def _w5(A, seed):
    return (np.random.default_rng(seed).standard_normal((A, H.HIDDEN)) * 0.05).astype(F32)


@pytest.mark.parametrize("rows", [1, 7, 8, 9, 33, 257])
@pytest.mark.parametrize("A", [1, 2, 17, 32])
def test_rules_within_fp32_bounds_of_float64(A, rows):
    h4, w5 = _h4(rows, rows + A), _w5(A, A)
    # rule 1: each product rounded once, then 5 butterfly sums and 16 warp sums on the way to Q
    q = H.q_rows(h4, w5)
    h64, w64 = h4.astype(np.float64), w5.astype(np.float64)
    exact = h64 @ w64.T
    bound = _gamma(1 + 5 + 16) * (np.abs(h64) @ np.abs(w64).T)
    assert (np.abs(q - exact) <= bound).all()
    assert q.dtype == F32 and q.shape == (rows, A)
    # rule 2: one product, ceil(rows / 8) running sums and three tree levels
    g = np.random.default_rng(rows * 31 + A)
    act = g.integers(0, A, rows)
    d = np.clip(g.standard_normal(rows), -1, 1).astype(F32)
    grad = H.fc2_grad(h4, d, act, A)
    onehot = np.zeros((rows, A))
    onehot[np.arange(rows), act] = d
    exact = onehot.T @ h64
    bound = _gamma(1 + -(-rows // 8) + 3) * (np.abs(onehot).T @ np.abs(h64))
    assert (np.abs(grad - exact) <= bound).all()
    assert grad.dtype == F32 and grad.shape == (A, H.HIDDEN)
    for a in set(range(A)) - set(act.tolist()):      # an action no row took has a zero gradient
        assert not grad[a].any()
    if rows == 1:                                     # one row: the product itself, rounded once
        assert (grad[act[0]] == (h4[0] * d[0]).astype(F32)).all()


def test_butterfly_against_lane_simulation():
    """Rule 1's vectorised butterfly against 32 scalar lanes exchanging values as __shfl_xor_sync does."""
    g = np.random.default_rng(5)
    vals = (g.standard_normal((50, 32)) * 10.0 ** g.integers(-3, 4, (50, 32))).astype(F32)
    got = H.butterfly(vals)
    for row, x in zip(vals, got):
        v = list(row)
        for o in (16, 8, 4, 2, 1):
            v = [F32(v[l] + v[l ^ o]) for l in range(32)]
        assert all(y == v[0] for y in v)              # every lane ends with the same sum
        assert x == v[0]


def test_q_rows_against_scalar_restatement():
    h4, w5 = _h4(3, 11), _w5(5, 12)
    q = H.q_rows(h4, w5)
    for b in range(3):
        for a in range(5):
            acc = F32(0)
            for w in range(16):
                lanes = [F32(h4[b, 32 * w + l] * w5[a, 32 * w + l]) for l in range(32)]
                for o in (16, 8, 4, 2, 1):
                    lanes = [F32(lanes[l] + lanes[l ^ o]) for l in range(32)]
                acc = F32(acc + lanes[0])
            assert q[b, a] == acc, (b, a)


def test_fc2_grad_against_scalar_restatement():
    rows, A = 19, 3
    h4 = _h4(rows, 13)
    g = np.random.default_rng(14)
    act, d = g.integers(0, A, rows), g.standard_normal(rows).astype(F32)
    grad = H.fc2_grad(h4, d, act, A)
    for a in range(A):
        for k in (0, 1, 100, 511):
            s = [F32(0)] * 8
            for b in range(rows):
                s[b % 8] = F32(s[b % 8] + (F32(h4[b, k] * d[b]) if act[b] == a else F32(0)))
            # k_opt_small: lane l holds s[l]; xor butterfly 1, 2, 4 leaves lane 0 with the tree
            for o in (1, 2, 4):
                s = [F32(s[l] + s[l ^ o]) for l in range(8)]
            assert grad[a, k] == s[0], (a, k)


def test_orders_are_observable():
    """A sequential row sum and a reversed warp order each give a different fp32 result on some element, so the GPU
    comparison can tell the device's orders from them."""
    h4, w5 = _h4(33, 21), _w5(17, 22)
    q = H.q_rows(h4, w5)
    assert (H.q_rows(h4, w5, warp_order=range(15, -1, -1)) != q).any()
    g = np.random.default_rng(23)
    act, d = g.integers(0, 2, 257), np.clip(g.standard_normal(257), -1, 1).astype(F32)
    parts = H.row_partials(_h4(257, 24), d, act, 2)
    assert (H.sequential(parts) != H.tree8(parts)).any()
    # at batch 33 and A = 32 most actions are taken by one or two rows; the orders still differ where three or more are
    act = g.integers(0, 32, 33)
    parts = H.row_partials(_h4(33, 25), np.clip(g.standard_normal(33), -1, 1).astype(F32), act, 32)
    assert (H.sequential(parts) != H.tree8(parts)).any()
