"""The Double DQN oracle (tests/double_oracle.py) against an independent torch-CPU autograd step that picks the
poststate action with torch.argmax, and its relation to the vanilla step."""
import numpy as np
import pytest
import torch

from double_oracle import DoubleDQNOracle, head_restated
from oracle import dqn_oracle as O
from test_oracle_dqn import torch_forward


def _batch(n, a, seed, terminal_p=0.3):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (n, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (n, 4, 84, 84)).astype(np.uint8)
    return (pre, rs.randint(0, a, n).astype(np.uint8), rs.randint(-3, 4, n).astype(np.int64), post,
            rs.rand(n) < terminal_p)


def _weights(a, seed):
    """Online and target weights that differ, with the last layers scaled so Q ~ O(1) like a trained net."""
    ws = O.xavier_init(a, seed=seed)
    tws = O.xavier_init(a, seed=seed + 100)
    for w in (ws, tws):
        w[3] *= np.float32(3)
        w[4] *= np.float32(3)
    return ws, tws


def _torch_double_step(ws, tws, mb, discount=0.99, clip=1.0):
    pre, act, rew, post, term = mb
    with torch.no_grad():
        tpost = torch_forward([torch.tensor(w) for w in tws], torch.tensor(post))
        astar = torch.argmax(torch_forward([torch.tensor(w) for w in ws], torch.tensor(post)), dim=1)
        chosen = tpost[torch.arange(len(astar)), astar].numpy()
    tw = [torch.tensor(w, requires_grad=True) for w in ws]
    preq = torch_forward(tw, torch.tensor(pre))
    r = np.clip(rew, -1, 1).astype(np.float64)
    y = np.where(term, r, r + discount * chosen.astype(np.float64)).astype(np.float32)
    pq = preq.detach().numpy()
    targets = pq.copy()
    targets[np.arange(len(act)), act] = y
    deltas = pq - targets
    cost = np.float32(np.mean(np.sum(np.square(deltas), axis=1) / 2))
    deltas = np.clip(deltas, -clip, clip)
    preq.backward(torch.tensor(deltas))
    return astar.numpy(), targets, cost, [t.grad.numpy() for t in tw]


@pytest.mark.parametrize("num_actions", [4, 18])
def test_double_oracle_matches_torch_argmax_step(num_actions):
    ws, tws = _weights(num_actions, 3)
    mb = _batch(16, num_actions, 1)
    orc = DoubleDQNOracle(num_actions, double_dqn=True, batch_size=16, weights=ws)
    for t, w in zip(orc.target_weights, tws):
        t[...] = w
    astar, targets, cost, grads = _torch_double_step(ws, tws, mb)
    orc.train(mb)
    L = orc.last
    assert (L["astar"] == astar).all()
    assert np.abs(L["targets"] - targets).max() <= 1e-5 * np.abs(targets).max()
    assert abs(L["cost"] - cost) <= 1e-5 * abs(cost)
    for g, ref in zip(L["grads"], grads):
        assert np.linalg.norm(g - ref) <= 1e-4 * np.linalg.norm(ref)
    # the online and target networks prefer different actions on some poststates, so the targets really differ
    assert (np.argmax(L["postq"], axis=1) != astar).any()


def _pair(num_actions, target_steps=10000, seed=5):
    ws, tws = _weights(num_actions, seed)
    a = O.DQNOracle(num_actions, batch_size=8, weights=ws, target_steps=target_steps)
    b = DoubleDQNOracle(num_actions, double_dqn=True, batch_size=8, weights=ws, target_steps=target_steps)
    return a, b, tws


def _same(a, b):
    assert a.last["cost"] == b.last["cost"]
    assert (a.last["deltas"] == b.last["deltas"]).all()
    for x, y in zip(a.weights, b.weights):
        assert (x == y).all()
    for x, y in zip(a.states, b.states):
        assert (x == y).all()


def test_double_equals_vanilla_at_target_steps_zero():
    a, b, _ = _pair(6, target_steps=0)
    for i in range(3):
        mb = _batch(8, 6, 10 + i)
        a.train(mb)
        b.train(mb)
        _same(a, b)


def test_double_equals_vanilla_right_after_target_sync():
    a, b, tws = _pair(6)
    for o in (a, b):
        for t, w in zip(o.target_weights, tws):
            t[...] = w
        o.update_target_network()
    mb = _batch(8, 6, 20)
    a.train(mb)
    b.train(mb)
    _same(a, b)


def test_double_target_differs_by_the_known_amount():
    """W5 rows built so the online network prefers action 1 and the target network action 0 on every state: the
    Double DQN target uses Q_target(s', 1) where the vanilla one uses Q_target(s', 0)."""
    ws, _ = _weights(2, 7)
    tws = [w.copy() for w in ws]
    h = np.abs(ws[4][0])
    ws[4][0], ws[4][1] = h, 2 * h                   # online: Q(s', 1) = 2 Q(s', 0) > 0
    tws[4][0], tws[4][1] = 3 * h, h                 # target: Q(s', 0) = 3 Q(s', 1)
    mb = _batch(8, 2, 30, terminal_p=0.0)
    pre, act, rew, post, term = mb
    qv = O.forward(tws, post)
    van = O.DQNOracle(2, batch_size=8, weights=ws)
    dbl = DoubleDQNOracle(2, double_dqn=True, batch_size=8, weights=ws)
    for o in (van, dbl):
        for t, w in zip(o.target_weights, tws):
            t[...] = w
        o.train(mb)
    assert (dbl.last["astar"] == 1).all() and (np.argmax(qv, axis=1) == 0).all()
    rows = np.arange(8)
    diff = van.last["targets"][rows, act].astype(np.float64) - dbl.last["targets"][rows, act]
    expect = 0.99 * (qv[:, 0].astype(np.float64) - qv[:, 1])
    assert np.abs(diff - expect).max() <= 1e-6 * np.abs(expect).max()
    assert (expect > 0).all()


def test_head_restatement_matches_oracle_targets():
    ws, tws = _weights(5, 9)
    mb = _batch(8, 5, 40)
    orc = DoubleDQNOracle(5, double_dqn=True, batch_size=8, weights=ws, clip_error=0)
    for t, w in zip(orc.target_weights, tws):
        t[...] = w
    orc.train(mb)
    L = orc.last
    deltas, row_cost = head_restated(L["preq"], L["postq"], L["online_postq"], mb[1], mb[2], mb[4], clip=0.0)
    assert (deltas == L["deltas"]).all()
    assert abs(np.float32(row_cost.mean()) - L["cost"]) <= 1e-6 * abs(L["cost"])
