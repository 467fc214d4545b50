"""The random-shift augmentation's rules (tests/shift_oracle.py) on the CPU: the clamp form against np.pad's
edge-replicate padding and a crop, the uniformity of the draws and the independence of the two slots, and the creation
refusals."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

import shift_oracle as SH


@pytest.mark.parametrize("pad", range(1, 9))
def test_clamp_form_is_edge_padding_and_crop(pad):
    """Every (dy, dx) in [-p, p]^2: the clamped gather equals np.pad(mode="edge") followed by the crop at (p + dy, p + dx),
    on frames whose every pixel differs from its neighbours."""
    rs = np.random.RandomState(pad)
    states = rs.randint(0, 256, (1, 2, 84, 84)).astype(np.uint8)
    for dy in range(-pad, pad + 1):
        for dx in range(-pad, pad + 1):
            off = np.array([[dy, dx]], np.int32)
            got = SH.shift(states, off)
            assert (got == SH.shift_padded(states, off, pad)).all(), (dy, dx)
            if dy == 0 and dx == 0:
                assert (got == states).all()


def test_draw_pins():
    """Known values: the offsets lie in [-p, p], counters and seeds change them, the (2, batch, 2) layout holds, and a
    batch's first rows do not depend on its size."""
    for pad in (1, 4, 8):
        d = SH.draw(7, 0, pad, 257)
        assert d.shape == (2, 257, 2) and d.dtype == np.int32
        assert d.min() >= -pad and d.max() <= pad
        assert (SH.draw(7, 0, pad, 32) == d[:, :32]).all()
        assert not (SH.draw(7, 1, pad, 257) == d).all()
        assert not (SH.draw(8, 0, pad, 257) == d).all()
    # the hash of rule 1 by hand for one entry, with Python integers
    m = (1 << 64) - 1

    def mix(x):
        x ^= x >> 30
        x = (x * 0xBF58476D1CE4E5B9) & m
        x ^= x >> 27
        x = (x * 0x94D049BB133111EB) & m
        return x ^ (x >> 31)
    seed, ctr, pad, z, b = 0xDEADBEEF12345678, 41, 4, 1, 13
    x = mix(mix((seed + 0x9E3779B97F4A7C15 * (ctr + 1)) & m) ^ (z << 32 | b))
    want = (((x >> 32) * (2 * pad + 1) >> 32) - pad, ((x & 0xFFFFFFFF) * (2 * pad + 1) >> 32) - pad)
    assert tuple(SH.draw(seed, ctr, pad, 16)[z, b]) == want


@pytest.mark.parametrize("pad", [1, 4, 8])
def test_draws_uniform_and_slots_independent(pad):
    """Over 200 counters x 512 samples: each slot's (dy, dx) is uniform over the (2p + 1)^2 cells (chi-square), and the
    two slots' offsets of the same sample are independent (chi-square test of the contingency table)."""
    k = 2 * pad + 1
    d = np.concatenate([SH.draw(0x1234567 + pad, c, pad, 512) for c in range(200)], axis=1)   # (2, 102400, 2)
    for z in range(2):
        cells = (d[z, :, 0] + pad) * k + (d[z, :, 1] + pad)
        counts = np.bincount(cells, minlength=k * k)
        assert stats.chisquare(counts).pvalue > 1e-4, (z, counts)
    for comp in range(2):   # dy of slot 0 against dy of slot 1, and the same for dx
        table = np.zeros((k, k), np.int64)
        np.add.at(table, (d[0, :, comp] + pad, d[1, :, comp] + pad), 1)
        assert stats.chi2_contingency(table)[1] > 1e-4, comp
    # and dy against dx within a slot
    table = np.zeros((k, k), np.int64)
    np.add.at(table, (d[0, :, 0] + pad, d[0, :, 1] + pad), 1)
    assert stats.chi2_contingency(table)[1] > 1e-4


def test_shift_seed_is_distinct_from_tau_seed():
    from simple_dqn_b200.deepqnetwork import shift_seed, tau_seed
    for s in (0, 1, 3, 7, 12345):
        assert shift_seed(s) != tau_seed(s)
        assert shift_seed(s) == shift_seed(s) and 0 <= shift_seed(s) < 1 << 64


def test_net_create_refuses_before_device_work():
    """random_shift outside 0..8 is EINVAL; the default is off."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.random_shift == 0 and cfg.shift_seed == 0
    for bad in (-1, 9, 84, -(1 << 31)):
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.random_shift = bad
        with pytest.raises(AssertionError, match="random_shift"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
