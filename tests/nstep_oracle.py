"""n-step returns (Hessel et al., 2018) on the CPU: a plain-Python restatement of the device's draw, window, return and
head (csrc/replay.cuh::sample_block, replay.cu::k_gather, per.cu::per_valid, net.cu::k_head), so that every index and
every head output compares bit for bit.  N = n_step, H = history_length, gamma = discount_rate.

Rules:
  1. Draw: index = random.randint(H, count - N), one MT19937 word per trial.  A trial is rejected when the window
     [index - H, index + N - 1] crosses the write pointer (index + N - 1 >= current and index - H < current) or when
     terminals[index - H : index] has a set flag.  count >= H + N.
  2. Minibatch: prestate getState(index - 1), action actions[index], poststate getState(index + N - 1), rewards and
     terminals of index .. index + N - 1.
  3. Return: c_k = min(max(float(rewards[index + k]), min_reward), max_reward); in fp64, g = 1; for k in 0..N-1:
     R = R + g * c_k; stop if terminals[index + k]; g = g * gamma.  Terminal: some flag in the window.
  4. Head: y = R if terminal, else R + g * Q^ with Q^ the maximum of the target row (or the target network's value at
     the first index of the maximum of the online network's poststate row); delta = preq[a] - float32(y); the row cost
     0.5 delta^2 before the clip, then the clip when clip > 0.  Every product and sum is one rounding (Python floats).
At N = 1 every rule is the reference's: oracle.replay_oracle.ReplayOracle and kernel_ref.head_td.
"""
import numpy as np

from oracle.mt19937 import MT19937

F32 = np.float32


def crosses_write_pointer(index, hist, n, current):
    """Rule 1's window test as the device writes it."""
    return index + n - 1 >= current and index - hist < current


def accept(ring, index, n):
    """Rule 1 for one trial on an oracle.replay_oracle.ReplayOracle."""
    h = ring.history_length
    if crosses_write_pointer(index, h, n, ring.current):
        return False
    return not ring.terminals[(index - h):index].any()


def valid_mask(terminals, count, current, hist, n):
    """Rule 1 for every slot of the ring: the leaves a prioritized ring may draw."""
    t = np.asarray(terminals).astype(bool)
    size = len(t)
    i = np.arange(size)
    cs = np.concatenate([[0], np.cumsum(t.astype(np.int64))])
    lo = np.clip(i - hist, 0, size)
    has_term = (cs[i] - cs[lo]) > 0
    return (i >= hist) & (i <= count - n) & ~((i + n - 1 >= current) & (i - hist < current)) & ~has_term


def sample_indexes(ring, rng: MT19937, n, batch=None):
    """Rule 1: (accepted indexes in acceptance order, MT19937 words consumed)."""
    h = ring.history_length
    assert ring.count >= h + n
    bs = ring.batch_size if batch is None else batch
    before = rng.words_drawn
    out = []
    while len(out) < bs:
        index = rng.randint(h, ring.count - n)
        if accept(ring, index, n):
            out.append(index)
    return np.array(out, dtype=np.int64), rng.words_drawn - before


def gather(ring, indexes, n):
    """Rule 2: (prestates, actions, (batch, N) rewards, poststates, (batch, N) terminals)."""
    pre = np.stack([ring.getState(i - 1) for i in indexes])
    post = np.stack([ring.getState(i + n - 1) for i in indexes])
    win = np.asarray(indexes, np.int64)[:, None] + np.arange(n)[None, :]
    return pre, ring.actions[indexes], ring.rewards[win], post, ring.terminals[win]


def clip_reward(r, min_reward, max_reward):
    return min(max(float(r), float(min_reward)), float(max_reward))


def n_step_return(rewards, terminals, discount, min_reward=-1, max_reward=1):
    """Rule 3 on one window: (R, g, terminal), g = gamma^N when no terminal."""
    R, g = 0.0, 1.0
    for r, t in zip(rewards, terminals):
        R = R + g * clip_reward(r, min_reward, max_reward)
        if t:
            return R, g, True
        g = g * float(discount)
    return R, g, False


def target(rewards, terminals, q_hat, discount, min_reward=-1, max_reward=1):
    """Rule 4's y in fp64."""
    R, g, term = n_step_return(rewards, terminals, discount, min_reward, max_reward)
    return R if term else R + g * float(q_hat)


def q_hat(postq, online_postq=None):
    """The target row's maximum, or (Double DQN) its value at the first index of the online row's maximum."""
    if online_postq is None:
        m = postq[0]
        for v in postq[1:]:
            m = max(m, v)
        return m
    best = 0
    for j in range(1, len(online_postq)):
        if online_postq[j] > online_postq[best]:
            best = j
    return postq[best]


def head_restated(preq, postq, actions, rewards, terminals, discount=0.99, min_reward=-1, max_reward=1, clip=1.0,
                  w=None, online_postq=None):
    """Rule 4 on the device's own fp32 Q rows and (batch, N) windows: (deltas, row costs, TD errors before the clip).
    w given: the prioritized step (the row cost and the clipped delta scaled by the importance weight)."""
    preq, postq = np.asarray(preq, F32), np.asarray(postq, F32)
    rewards, terminals = np.asarray(rewards), np.asarray(terminals)
    if rewards.ndim == 1:
        rewards, terminals = rewards[:, None], terminals[:, None]
    b, A = preq.shape
    deltas = np.zeros((b, A), F32)
    row_cost = np.zeros(b, F32)
    td = np.zeros(b, F32)
    for i in range(b):
        q = q_hat(postq[i], None if online_postq is None else online_postq[i])
        y = target(rewards[i], terminals[i], q, discount, min_reward, max_reward)
        a = actions[i]
        d = F32(preq[i, a] - F32(y))
        td[i] = d
        wi = F32(1) if w is None else F32(w[i])
        row_cost[i] = F32(0.5) * d * d if w is None else wi * (F32(0.5) * d * d)
        if clip > 0:
            d = F32(min(max(d, F32(-clip)), F32(clip)))
        deltas[i, a] = d if w is None else d * wi
    return deltas, row_cost, td


def train_step(net, minibatch, double=False):
    """oracle.dqn_oracle.DQNOracle.train with the n-step target (rule 4, Q^ of the target network on the poststates)
    on a gathered (batch, N) minibatch: the numpy trajectory oracle extended with the n-step return."""
    from oracle import dqn_oracle as O
    prestates, actions, rewards, poststates, terminals = minibatch
    postq = O.forward(net.target_weights, poststates)
    online_post = O.forward(net.weights, poststates) if double else None
    preq, acts = O.forward(net.weights, prestates, keep=True)
    targets = preq.copy()
    for i, a in enumerate(actions):
        q = q_hat(postq[i], None if online_post is None else online_post[i])
        targets[i, a] = F32(target(rewards[i], terminals[i], q, net.discount_rate, net.min_reward, net.max_reward))
    deltas = preq - targets
    cost = F32(np.mean(np.sum(np.square(deltas), axis=1) / F32(2.0)))
    if net.clip_error:
        deltas = np.clip(deltas, -net.clip_error, net.clip_error)
    grads = O.backward(net.weights, acts, deltas)
    assert net.optimizer == "rmsprop"
    O.rmsprop_update(net.weights, net.states, grads, prestates.shape[0], net.learning_rate, net.decay_rate)
    net.train_iterations += 1
    return cost
