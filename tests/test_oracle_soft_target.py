"""The soft target update's restatement (tests/soft_target_oracle.py) against a float64 reference, its end points, and the
refusals of b200dqn_net_create and the manual entry that happen before any device work (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest

import soft_target_oracle as SOFT

F32 = np.float32


def _ulp(a):
    """float32 ulp at |a| (float64 values rounded to float32 first), elementwise, as float64."""
    return np.spacing(np.abs(np.asarray(a, np.float64).astype(F32))).astype(np.float64)


@pytest.mark.parametrize("tau", [0.005, 0.01, 0.1, 0.5, 0.999, 1e-6, 1.0 / 3.0])
def test_restatement_against_float64(tau):
    """fl(fl(c x) + fl(t y)) against the exact c x + t y (float64, the same float32 factors, which are float32(1 - tau)
    and float32(tau)).  Same-signed operands keep the sum free of cancellation: there the error is within half an ulp
    of each of the three roundings, (ulp(c x) + ulp(t y) + ulp(sum)) / 2, which is one ulp of the result plus the
    product roundings' excess where the sum sits just above a power of two (1.25 ulp at most here).  Every element,
    mixed signs included, equals the explicit model of three separately rounded float64 operations bit for bit."""
    rs = np.random.RandomState(int(tau * 1e6) % 1000)
    x = (rs.randn(200000) * 0.05).astype(F32)
    y = (x + rs.randn(200000).astype(F32) * F32(1e-3)).astype(F32)
    c, t = SOFT.factors(tau)
    assert c == F32(1.0 - tau) and t == F32(tau)
    got = SOFT.blend(x, y, tau)
    assert got.dtype == F32
    p1 = np.float64(c) * x.astype(np.float64)
    p2 = np.float64(t) * y.astype(np.float64)
    exact = p1 + p2
    same = np.sign(x) == np.sign(y)
    err = np.abs(got.astype(np.float64) - exact)
    bound = (_ulp(p1) + _ulp(p2) + _ulp(exact)) / 2
    assert (err[same] <= bound[same]).all()
    assert (err[same] <= 1.25 * _ulp(exact)[same]).all()
    # every operation rounded on its own: the float64 products and sum of float32 values, each rounded to float32
    model = (np.float64(c) * x.astype(np.float64)).astype(F32).astype(np.float64) + \
            (np.float64(t) * y.astype(np.float64)).astype(F32).astype(np.float64)
    assert (got.view(np.uint32) == model.astype(F32).view(np.uint32)).all()


def test_factors_form_one_minus_tau_in_float64():
    """c is float32(1 - tau) with 1 - tau formed in float64, not 1 - float32(tau)."""
    tau = 0.005
    c, t = SOFT.factors(tau)
    assert c == F32(1.0 - 0.005) and t == F32(0.005)
    # a tau whose float32 rounding moves 1 - tau: the float64 difference is what the rule rounds
    tau = 1.0 - 2.0 ** -30
    assert SOFT.factors(tau)[0] == F32(2.0 ** -30) != F32(F32(1) - F32(tau))


def test_tau_one_and_tau_zero():
    """tau = 1 gives the online weights, tau = 0 keeps the target (in value: a signed zero may flip)."""
    rs = np.random.RandomState(1)
    x = rs.randn(10000).astype(F32)
    y = rs.randn(10000).astype(F32)
    assert (SOFT.blend(x, y, 1.0) == y).all()
    assert (SOFT.blend(x, y, 1.0).view(np.uint32) == y.view(np.uint32)).all()   # no zeros among them
    assert (SOFT.blend(x, y, 0.0) == x).all()
    assert (SOFT.blend(x, y, 0.0).view(np.uint32) == x.view(np.uint32)).all()
    layers = SOFT.blend_layers([x, y], [y, x], 1.0)
    assert (layers[0] == y).all() and (layers[1] == x).all()


def test_repeated_blends_converge_to_the_online_weights():
    """k blends at tau leave (1 - tau)^k of the gap, to float32 accuracy."""
    rs = np.random.RandomState(2)
    x = rs.randn(1000).astype(F32)
    y = rs.randn(1000).astype(F32)
    tw = x
    for _ in range(200):
        tw = SOFT.blend(tw, y, 0.05)
    gap = (1 - 0.05) ** 200
    assert np.abs(tw.astype(np.float64) - (y + gap * (x.astype(np.float64) - y))).max() < 1e-5


def _cfg(**kw):
    from simple_dqn_b200 import _lib as L
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def test_config_default_is_off():
    assert _cfg().soft_target_tau == 0.0


@pytest.mark.parametrize("kw", [{"soft_target_tau": -0.1}, {"soft_target_tau": 1.5}, {"soft_target_tau": math.nan},
                                {"soft_target_tau": math.inf}, {"soft_target_tau": -math.inf},
                                {"soft_target_tau": -0.0001},
                                {"soft_target_tau": 0.005, "target_steps": 0},
                                {"soft_target_tau": 1.0, "target_steps": 0}])
def test_net_create_refuses_before_device_work(kw):
    """A tau outside [0, 1], a non-finite tau, and tau > 0 with target_steps = 0 are EINVAL before any device work, on
    both engines."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    for mode in (L.MATH_FP32_SIMT, L.MATH_TCGEN05):
        cfg = _cfg(math_mode=mode, **kw)
        with pytest.raises(AssertionError, match="soft"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))


def test_deepqnetwork_refuses_before_device_work():
    from helpers import make_args
    from simple_dqn_b200 import DeepQNetwork
    for kw in ({"soft_target_tau": 2.0}, {"soft_target_tau": 0.01, "target_steps": 0}):
        with pytest.raises(AssertionError, match="soft"):
            DeepQNetwork(4, make_args(**kw))


def test_manual_entry_refuses_a_null_net():
    from simple_dqn_b200 import _lib as L
    with pytest.raises(AssertionError):
        L.call("b200dqn_net_soft_update_target", None, 0.5, None)
