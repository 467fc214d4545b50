"""tests/dueling_oracle.py against independent computations (CPU): the head's and the whole network's gradients against
torch autograd of sum huber(delta) through V + (A - mean A), the forward within fp32 bounds of float64, the A = 1 edge,
the Xavier draw, and the dueling arguments net_create refuses before any device work."""
import ctypes as C

import numpy as np
import pytest
import torch

import dueling_oracle as D
import head_oracle as H

F32 = np.float32
EPS = float(np.finfo(F32).eps)


def _head_case(A, rows, seed):
    g = np.random.default_rng(seed)
    z4 = g.standard_normal((rows, 1024)).astype(F32)
    w5 = (g.standard_normal((A + 1, 512)) * 0.05).astype(F32)
    return z4, np.maximum(z4, F32(0)), w5, g.integers(0, A, rows), g.standard_normal(rows).astype(F32)


@pytest.mark.parametrize("A", [1, 2, 5, 17, 32])
def test_head_gradients_match_autograd(A):
    """dZ4 and dW5 of rule 3 / 4 against torch autograd (float64) of sum_b huber(Q[b, a_b] - y_b), clip 1."""
    z4, h4, w5, act, y = _head_case(A, 37, A)
    q = D.q_rows(h4, w5)
    d = np.clip(q[np.arange(37), act] - y, F32(-1), F32(1)).astype(F32)
    dA, dV = D.stream_grads(d, act, A)
    tz = torch.tensor(z4, dtype=torch.float64, requires_grad=True)
    tw = torch.tensor(w5, dtype=torch.float64, requires_grad=True)
    th = torch.relu(tz)
    adv = th[:, :512] @ tw[:A].T
    val = th[:, 512:] @ tw[A]
    tq = val[:, None] + adv - adv.mean(dim=1, keepdim=True)
    sel = tq[torch.arange(37), torch.tensor(act)]
    torch.nn.functional.huber_loss(sel, torch.tensor(y, dtype=torch.float64), reduction="sum", delta=1.0).backward()
    got_dz, got_dw = D.dz4(h4, w5, dA, dV), D.fc2_grad(h4, dA, dV)
    for got, ref in ((got_dz, tz.grad.numpy()), (got_dw, tw.grad.numpy())):
        assert np.abs(got - ref).max() <= 1e-5 * np.abs(ref).max(), np.abs(got - ref).max()
    assert (got_dz[h4 <= 0] == 0).all()


@pytest.mark.parametrize("A", [1, 2, 17, 32])
@pytest.mark.parametrize("rows", [1, 33, 257])
def test_forward_within_fp32_bounds_of_float64(A, rows):
    """Rules 1 and 2 against float64: every error inside a bound of the fp32 roundings of its terms."""
    _, h4, w5, _, _ = _head_case(A, rows, 100 + A)
    adv, val = D.streams(h4, w5)
    q = D.aggregate(adv, val)
    h, w = h4.astype(np.float64), w5.astype(np.float64)
    adv64 = h[:, :512] @ w[:A].T
    val64 = h[:, 512:] @ w[A]
    q64 = val64[:, None] + adv64 - adv64.mean(axis=1, keepdims=True)
    sa = np.abs(h[:, :512]) @ np.abs(w[:A]).T
    sv = np.abs(h[:, 512:]) @ np.abs(w[A])
    assert (np.abs(adv - adv64) <= 64 * EPS * sa).all()
    assert (np.abs(val - val64) <= 64 * EPS * sv).all()
    bound = 128 * EPS * (sv[:, None] + sa + sa.max(axis=1, keepdims=True))
    assert (np.abs(q - q64) <= bound).all()


def test_one_action_is_the_value_stream():
    """A = 1: Q = V exactly, and the advantage gradient (dA, fc2's advantage row, dZ4 on the advantage units) is exactly
    zero."""
    _, h4, w5, act, _ = _head_case(1, 33, 7)
    adv, val = D.streams(h4, w5)
    assert (D.aggregate(adv, val)[:, 0] == val).all()
    d = np.random.default_rng(1).standard_normal(33).astype(F32)
    dA, dV = D.stream_grads(d, act, 1)
    assert (dA == 0).all() and not np.signbit(dA).any()
    assert (D.fc2_grad(h4, dA, dV)[0] == 0).all()
    assert (D.dz4(h4, w5, dA, dV)[:, :512] == 0).all()


def test_rules_tell_wrong_variants_apart():
    """The restated rules differ from the variants a faulty head would compute: no mean subtracted, the mean over
    A + 1, dA without its -delta/A term."""
    _, h4, w5, act, _ = _head_case(6, 33, 9)
    adv, val = D.streams(h4, w5)
    q = D.aggregate(adv, val)
    assert (q != D.aggregate(adv, val, skip_mean=True)).any()
    assert (q != D.aggregate(adv, val, mean_div=7)).any()
    d = np.random.default_rng(2).standard_normal(33).astype(F32)
    assert (D.stream_grads(d, act, 6)[0] != D.stream_grads(d, act, 6, drop_mean_term=True)[0]).any()
    assert (H.q_rows(h4[:, :512], w5[:6]) == adv).all()


def _torch_net(weights, states):
    """Float64 torch forward of the whole dueling network from Neon-layout weights: (rows, A) Q."""
    x = torch.tensor(states, dtype=torch.float64) / 255.0
    for li, (r, st) in enumerate(((8, 4), (4, 2), (3, 1))):
        k = weights[li].shape[1]
        x = torch.relu(torch.nn.functional.conv2d(x, weights[li].T.reshape(k, -1, r, r), stride=st))
    h4 = torch.relu(x.reshape(len(x), -1) @ weights[3].T)
    A = weights[4].shape[0] - 1
    adv = h4[:, :512] @ weights[4][:A].T
    val = h4[:, 512:] @ weights[4][A]
    return val[:, None] + adv - adv.mean(dim=1, keepdim=True)


@pytest.mark.parametrize("double", [False, True], ids=["vanilla", "double"])
@pytest.mark.parametrize("A", [1, 4])
def test_whole_network_step_matches_autograd(A, double):
    """numpy_step's gradients of every layer against torch autograd of the cost (sum of 0.5 delta^2 with the clip as
    huber, i.e. the reference's clipped-delta backward) through the whole dueling network, float64."""
    rows = 4
    g = np.random.default_rng(A + 10 * double)
    ws = D.xavier_init(A, 5)
    ws[3] *= F32(3)
    ws[4] *= F32(3)
    tw = [(w + (g.standard_normal(w.shape) * 0.1 * np.abs(w).max())).astype(F32) for w in ws]
    pre = g.integers(0, 256, (rows, 4, 84, 84)).astype(np.uint8)
    post = g.integers(0, 256, (rows, 4, 84, 84)).astype(np.uint8)
    act = g.integers(0, A, rows)
    rew = g.integers(-2, 3, rows)
    term = np.array([0, 1, 0, 0], np.uint8)
    mb = (pre, act, rew, post, term)
    w_np = [w.copy() for w in ws]
    _, grads = D.numpy_step(w_np, [np.zeros_like(w) for w in ws], tw, mb, double=double)
    # the target, in float64 from the numpy forward (it carries no gradient)
    postq = D.forward(tw, post).astype(np.float64)
    pick = np.argmax(D.forward(ws, post), axis=1) if double else np.argmax(postq, axis=1)
    y = np.clip(rew, -1, 1) + 0.99 * postq[np.arange(rows), pick] * (1 - term)
    tws = [torch.tensor(w, dtype=torch.float64, requires_grad=True) for w in ws]
    q = _torch_net(tws, pre)
    sel = q[torch.arange(rows), torch.tensor(act)]
    torch.nn.functional.huber_loss(sel, torch.tensor(y), reduction="sum", delta=1.0).backward()
    for l in range(5):
        ref = tws[l].grad.numpy()
        assert np.linalg.norm(grads[l] - ref) <= 1e-4 * np.linalg.norm(ref), l


def test_xavier_shapes_and_draw_order():
    """Dueling shapes (1024, 3136) and (A + 1, 512), drawn from one RandomState in layer order: the conv layers are
    the scalar net's draws, and fc1 / fc2 continue the same stream."""
    from oracle import dqn_oracle as O
    ws = D.xavier_init(4, 3)
    assert [w.shape for w in ws] == [(256, 32), (512, 64), (576, 64), (1024, 3136), (5, 512)]
    base = O.xavier_init(4, 3)
    for l in range(3):
        assert (ws[l] == base[l]).all()
    rng = np.random.RandomState(3)
    for shp in [(256, 32), (512, 64), (576, 64)]:
        rng.uniform(-1, 1, shp)
    s = np.sqrt(3.0 / 3136)
    assert (ws[3] == rng.uniform(-s, s, (1024, 3136)).astype(F32)).all()
    assert np.abs(ws[3]).max() <= s and np.abs(ws[4]).max() <= np.sqrt(3.0 / 512)


def test_net_create_refuses_before_device_work():
    """dueling outside {0, 1} is EINVAL; with a distributional head it is ENOTIMPL."""
    from simple_dqn_b200 import _lib as L
    h = C.c_void_p()
    cfg = L.NetConfig()
    L.call("b200dqn_net_config_default", C.byref(cfg), 4)
    assert cfg.dueling == 0
    for bad, exc, fields in ((2, AssertionError, {}), (-1, AssertionError, {}),
                             (1, NotImplementedError, {"num_atoms": 51})):
        L.call("b200dqn_net_config_default", C.byref(cfg), 4)
        cfg.dueling = bad
        for k, v in fields.items():
            setattr(cfg, k, v)
        with pytest.raises(exc, match="dueling"):
            L.call("b200dqn_net_create", 0, C.byref(cfg), C.byref(h))
