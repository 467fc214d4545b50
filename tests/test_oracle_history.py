"""The numpy oracle at history lengths other than 4, cross-checked against the torch-CPU restatement.

The network takes the H frames of a state as conv1's input channels (deepqnetwork.py:37), so conv1 has
64*H filter rows and every later layer keeps its shape.  Same bars as tests/test_oracle_dqn.py."""
import numpy as np
import pytest
import torch

from oracle import dqn_oracle as O
from oracle.dqn_torch import TorchDQN

HISTS = [1, 3, 8]


def _batch(n, hist, a, seed):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8)
    return pre, rs.randint(0, a, n).astype(np.uint8), rs.randint(-3, 4, n).astype(np.int64), post, rs.rand(n) < 0.3


@pytest.mark.parametrize("hist", HISTS)
def test_shapes_follow_history_length(hist):
    shp = O.layer_shapes(4, history_length=hist)
    assert shp == [(64 * hist, 32), (512, 64), (576, 64), (512, 3136), (4, 512)]
    ws = O.xavier_init(4, seed=3, history_length=hist)
    assert [w.shape for w in ws] == shp
    bound = np.sqrt(3.0 / (64 * hist))                         # Xavier(local=True): fan_in = C*R*S
    assert np.abs(ws[0]).max() <= bound and np.abs(ws[0]).max() > 0.9 * bound


@pytest.mark.parametrize("hist", HISTS)
def test_forward_backward_match_torch_autograd(hist):
    ws = O.xavier_init(6, seed=3, history_length=hist)
    pre, *_ = _batch(8, hist, 6, 0)
    q, acts = O.forward(ws, pre, keep=True)
    tw = [torch.tensor(w, requires_grad=True) for w in ws]
    tq = TorchDQN._forward(tw, torch.tensor(pre))
    assert np.abs(tq.detach().numpy() - q).max() <= 1e-5 * np.abs(q).max()
    d = np.random.RandomState(1).randn(8, 6).astype(np.float32)
    tq.backward(torch.tensor(d))
    for g, t in zip(O.backward(ws, acts, d), tw):
        ref = t.grad.numpy()
        assert g.shape == ref.shape
        assert np.linalg.norm(g - ref) <= 1e-4 * np.linalg.norm(ref)


@pytest.mark.parametrize("hist", HISTS)
def test_train_step_matches_torch(hist):
    ws = O.xavier_init(4, seed=5, history_length=hist)
    ws[3] = ws[3] * np.float32(3.0)                            # Q ~ O(1), as in the GPU parity tests
    ws[4] = ws[4] * np.float32(3.0)
    orc = O.DQNOracle(4, batch_size=8, weights=ws)
    tor = TorchDQN(ws)
    mb = _batch(8, hist, 4, 2)
    cost = orc.train(mb)
    tcost = tor.train(mb)
    assert abs(cost - tcost) <= 1e-5 * abs(tcost)
    for l in range(5):
        upd, tupd = orc.weights[l] - ws[l], tor.w[l].numpy() - ws[l]
        assert np.linalg.norm(upd - tupd) <= 1e-3 * np.linalg.norm(tupd), l
