"""Global gradient-norm clipping's restatement (tests/grad_clip_oracle.py) against torch.nn.utils.clip_grad_norm_, its
identity for a large max_grad_norm, and the refusals that happen before any device work (no GPU needed)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import grad_clip_oracle as CLIP
from oracle import dqn_oracle as O

F32 = np.float32


def _grads(seed, iqn, scale):
    rs = np.random.RandomState(seed)
    shapes = O.layer_shapes(4) + ([(3136, 64)] if iqn else [])
    return [(rs.randn(*s) * scale).astype(F32) for s in shapes]


@pytest.mark.parametrize("iqn", [False, True])
@pytest.mark.parametrize("max_norm", [1e-3, 0.5, 10.0])
@pytest.mark.parametrize("bsz", [1, 32, 257])
def test_restatement_matches_torch_clip_grad_norm(iqn, max_norm, bsz):
    """On random gradients at the real layer shapes, c32 and gg' agree with clip_grad_norm_ on the same g / bsz: in
    float64 to the float32 rounding of c32 and gg', in float32 up to the rounding of torch's float32 norm."""
    grads = _grads(bsz + (7 if iqn else 0), iqn, 0.3 * bsz)
    got, sq, n, c = CLIP.clip(grads, bsz, max_norm)
    assert len(sq) == 6 and (sq[5] == 0.0) != iqn
    assert c < 1
    for dtype, tol in ((torch.float64, 2.0 ** -23), (torch.float32, 1e-4)):
        params = [torch.nn.Parameter(torch.zeros(g.shape, dtype=dtype)) for g in grads]
        for p, g in zip(params, CLIP.scaled_grads(grads, bsz)):
            p.grad = torch.from_numpy(g.copy()).to(dtype)
        tn = float(torch.nn.utils.clip_grad_norm_(params, max_norm))
        assert abs(tn - n) <= tol * n
        tc = max_norm / (tn + 1e-6)
        assert abs(float(c) - tc) <= 2 * tol * tc
        for p, g in zip(params, got):
            ref = p.grad.numpy().astype(np.float64)
            assert (np.abs(g - ref) <= 3 * tol * np.abs(ref)).all(), np.abs(g - ref).max()


@pytest.mark.parametrize("bsz", [1, 32])
def test_a_large_max_norm_is_the_identity(bsz):
    grads = _grads(3, True, 1.0)
    got, _, n, c = CLIP.clip(grads, bsz, 1e30)
    assert c == F32(1.0) and n > 0
    for g, x in zip(got, CLIP.scaled_grads(grads, bsz)):
        assert (g.view(np.uint32) == x.view(np.uint32)).all()


def test_nan_and_infinite_norms():
    """A NaN norm leaves the gradients alone (c32 = 1), as clipping never happened; an infinite norm gives c32 = 0."""
    assert CLIP.clip_scale(math.nan, 10.0) == F32(1.0)
    assert CLIP.clip_scale(math.inf, 10.0) == F32(0.0)
    assert CLIP.clip_scale(0.0, 10.0) == F32(1.0)


def test_sum_of_squares_is_exact_products():
    """Every square of a float32 value is exact in float64, so S_l is only rounded by the sum."""
    x = np.array([1.0 + 2.0 ** -23, 3.0 * 2.0 ** -140, -7.5], F32)
    assert CLIP.layer_sq(x) == math.fsum([float(v) * float(v) for v in x])


def _cfg(**kw):
    from simple_dqn_b200 import _lib as L
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def test_config_default_is_off():
    assert _cfg().max_grad_norm == 0.0


@pytest.mark.parametrize("bad", [-1.0, -1e-30, math.nan, math.inf, -math.inf])
def test_net_create_refuses_before_device_work(bad):
    """A negative, NaN or infinite max_grad_norm is EINVAL before any device work, on both engines."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    for mode in (L.MATH_FP32_SIMT, L.MATH_TCGEN05):
        with pytest.raises(AssertionError, match="max_grad_norm"):
            L.call("b200dqn_net_create", 0, C.byref(_cfg(math_mode=mode, max_grad_norm=bad)), C.byref(h))


def test_deepqnetwork_refuses_before_device_work():
    from helpers import make_args
    from simple_dqn_b200 import DeepQNetwork
    with pytest.raises(AssertionError, match="max_grad_norm"):
        DeepQNetwork(4, make_args(max_grad_norm=-10.0))


def test_selectors_are_appended():
    from simple_dqn_b200 import _lib as L
    assert (L.NET_PTR_BOOT_ACTIVE_HEAD, L.NET_PTR_GRAD_SQ, L.NET_PTR_GRAD_NORM, L.NET_PTR_CLIP_SCALE) == (53, 54, 55, 56)
    assert L.NetConfig._fields_[-1] == ("max_grad_norm", C.c_double)
