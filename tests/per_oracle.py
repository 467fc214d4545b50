"""Proportional prioritized experience replay (Schaul et al., 2016; OpenAI baselines' PrioritizedReplayBuffer) on the
CPU: a numpy restatement of the device's trees, draw, importance weights and weighted train step (csrc/per.cu,
k_head), with the device's node layout and summation order, so that every node and every draw compares bit for bit.

Rules:
  1. Leaf i of the sum tree is the stored priority of slot i if getMinibatch would accept i as an index
     (hist <= i <= count - 1, not i in [current, current + hist), no terminal in terminals[i-hist .. i-1]), else 0.
  2. Stored priorities are p^alpha in fp64: max_priority^alpha for a written slot, (|delta| + eps)^alpha after a step
     (the last occurrence of a repeated slot wins); max_priority = max(max_priority, |delta| + eps), from 1.
  3. The tree is 32-ary, level by level; a node is its 32 children reduced by an xor butterfly (16, 8, 4, 2, 1).  A
     draw takes mass_i = random.random() * (total / batch) + i * (total / batch) and descends: at each node the
     first child whose inclusive prefix sum (warp scan: Hillis-Steele, 1, 2, 4, 8, 16) exceeds the mass, else the
     last child with a positive sum; the mass loses the prefix before the chosen child.
  4. w_i = (N P_i)^-beta / (N P_min)^-beta, P = leaf / total, N = count, beta = beta0 + (1 - beta0) min(1, k / steps)
     with k the samplings done, in fp64, rounded once to fp32.
  5. The head scales the clipped delta by w_i and the per-row cost (taken before the clip) by w_i.
"""
import numpy as np

from oracle import dqn_oracle as O
from oracle.mt19937 import MT19937

F32 = np.float32
INF = np.float64(np.inf)


def valid_mask(terminals, count, current, hist):
    """Rule 1 for every slot of the ring."""
    t = np.asarray(terminals).astype(bool)
    size = len(t)
    i = np.arange(size)
    cs = np.concatenate([[0], np.cumsum(t.astype(np.int64))])
    lo = np.clip(i - hist, 0, size)
    has_term = (cs[i] - cs[lo]) > 0
    return (i >= hist) & (i <= count - 1) & ~((i >= current) & (i - hist < current)) & ~has_term


def layout(size):
    """(nodes per level, start of each level): level 0 holds the leaves, every level starts at a multiple of 32."""
    n = [int(size)]
    while n[-1] > 1:
        n.append((n[-1] + 31) // 32)
    off = [0]
    for x in n:
        off.append(off[-1] + (x + 31) // 32 * 32)
    return n, off


def _pad32(x, fill):
    m = (len(x) + 31) // 32 * 32
    out = np.full(m, fill, dtype=np.float64)
    out[:len(x)] = x
    return out


def butterfly(x, op):
    """x (m, 32) -> (m,): lane 0 of the warp's xor butterfly 16, 8, 4, 2, 1."""
    x = np.asarray(x, np.float64)
    for o in (16, 8, 4, 2, 1):
        x = op(x[:, :o], x[:, o:2 * o])
    return x[:, 0]


def parent_level(child, fill, op):
    return butterfly(_pad32(child, fill).reshape(-1, 32), op)


def build(leaves):
    """Sum levels and min levels (min level 0 = leaf if positive else +inf) of the tree over `leaves`."""
    leaves = np.asarray(leaves, np.float64)
    sums = [leaves]
    mins = [np.where(leaves > 0, leaves, INF)]
    while len(sums[-1]) > 1:
        sums.append(parent_level(sums[-1], 0.0, np.add))
        mins.append(parent_level(mins[-1], INF, np.minimum))
    return sums, mins


def internal_from_leaves(leaves):
    """Every node above the leaves, given the leaves: what the device must hold over its own leaves."""
    return build(leaves)


def flat_sum(sums):
    """The device's SUM_TREE layout."""
    return np.concatenate([_pad32(s, 0.0) for s in sums])


def split_flat(flat, size, minimum=False):
    """Device SUM_TREE (or MIN_TREE, levels 1..) -> list of levels without their padding."""
    n, off = layout(size)
    if minimum:
        return [flat[off[l] - off[1]:off[l] - off[1] + n[l]] for l in range(1, len(n))]
    return [flat[off[l]:off[l] + n[l]] for l in range(len(n))]


def random_from_words(w0, w1):
    """CPython's random.random() from two MT19937 output words."""
    return ((w0 >> 5) * 67108864.0 + (w1 >> 6)) * (1.0 / 9007199254740992.0)


def scan_inclusive(x):
    """The warp's Hillis-Steele inclusive scan (offsets 1, 2, 4, 8, 16)."""
    x = np.asarray(x, np.float64).copy()
    for o in (1, 2, 4, 8, 16):
        y = x.copy()
        y[o:] = x[o:] + x[:-o]
        x = y
    return x


def descend(sums, mass):
    """Rule 3 for one mass: (slot, leaf value)."""
    node = 0
    leaf = 0.0
    for l in range(len(sums) - 2, -1, -1):
        x = _pad32(sums[l], 0.0)[node * 32:node * 32 + 32]
        incl = scan_inclusive(x)
        gt = np.nonzero(incl > mass)[0]
        if len(gt):
            pick = int(gt[0])
        else:
            pos = np.nonzero(x > 0)[0]
            pick = int(pos[-1]) if len(pos) else 0
        if pick > 0:
            mass = mass - incl[pick - 1]
        leaf = float(x[pick])
        node = node * 32 + pick
    return node, leaf


def beta_at(k, beta0, beta_steps):
    frac = min(1.0, k / beta_steps) if beta_steps > 0 else 1.0
    return beta0 + (1.0 - beta0) * frac


def weight(leaf, total, minv, count, beta):
    return F32(((count * (leaf / total)) ** -beta) / ((count * (minv / total)) ** -beta))


def draw(sums, mins, rng: MT19937, batch, count, k=0, beta0=0.4, beta_steps=1.0):
    """A stratified draw of `batch` indexes (rule 3) and their weights (rule 4); advances rng by 2 * batch words."""
    total = float(sums[-1][0])
    assert total > 0
    minv = float(mins[-1][0])
    seg = total / batch
    beta = beta_at(k, beta0, beta_steps)
    idx = np.zeros(batch, np.int64)
    w = np.zeros(batch, F32)
    for i in range(batch):
        w0 = rng.genrand_uint32()
        w1 = rng.genrand_uint32()
        mass = random_from_words(w0, w1) * seg + float(i) * seg
        idx[i], leaf = descend(sums, mass)
        w[i] = weight(leaf, total, minv, float(count), beta)
    return idx, w


class PEROracle:
    """Priorities and trees of one ring (the ring itself: oracle.replay_oracle.ReplayOracle)."""

    def __init__(self, ring, alpha=0.6, beta0=0.4, beta_steps=1.0, eps=1e-6):
        self.ring = ring
        self.alpha, self.beta0, self.beta_steps, self.eps = alpha, beta0, beta_steps, eps
        self.prio = np.ones(ring.size, np.float64)
        self.max_priority = 1.0
        self.samplings = 0

    def add(self, action, reward, screen, terminal):
        self.prio[self.ring.current] = self.max_priority ** self.alpha
        self.ring.add(action, reward, screen, terminal)

    def leaves(self):
        r = self.ring
        return np.where(valid_mask(r.terminals, r.count, r.current, r.history_length), self.prio, 0.0)

    def tree(self):
        return build(self.leaves())

    def draw(self, rng, batch=None):
        sums, mins = self.tree()
        out = draw(sums, mins, rng, batch or self.ring.batch_size, self.ring.count, self.samplings, self.beta0,
                   self.beta_steps)
        self.samplings += 1
        return out

    def weights_of(self, idx):
        sums, mins = self.tree()
        beta = beta_at(self.samplings, self.beta0, self.beta_steps)
        return np.array([weight(self.prio[i], float(sums[-1][0]), float(mins[-1][0]), float(self.ring.count), beta)
                         for i in idx], F32)

    def update(self, idx, td_err):
        for i, d in zip(idx, td_err):      # sequential: the last occurrence wins
            a = abs(float(d)) + self.eps
            self.prio[i] = a ** self.alpha
            self.max_priority = max(self.max_priority, a)


def head_restated(preq, postq, actions, rewards, terminals, w, discount=0.99, min_reward=-1, max_reward=1, clip=1.0,
                  online_postq=None):
    """k_head's weighted TD step on given fp32 Q rows, bit for bit: (deltas, row costs, TD errors before the clip).
    online_postq given: the Double DQN target (first index of its maximum)."""
    r = np.clip(rewards, min_reward, max_reward)
    n, A = preq.shape
    deltas = np.zeros((n, A), F32)
    row_cost = np.zeros(n, F32)
    td = np.zeros(n, F32)
    for i in range(n):
        if online_postq is None:
            maxq = postq[i, 0]
            for j in range(1, A):
                maxq = max(maxq, postq[i, j])
        else:
            best = 0
            for j in range(1, A):
                if online_postq[i, j] > online_postq[i, best]:
                    best = j
            maxq = postq[i, best]
        y = float(r[i]) if terminals[i] else float(r[i]) + discount * float(maxq)
        d = F32(preq[i, actions[i]] - F32(y))
        td[i] = d
        row_cost[i] = F32(w[i]) * (F32(0.5) * d * d)
        if clip > 0:
            d = F32(min(max(d, F32(-clip)), F32(clip)))
        deltas[i, actions[i]] = d * F32(w[i])
    return deltas, row_cost, td


def train_weighted(net: O.DQNOracle, minibatch, w):
    """DQNOracle.train with rule 5: the per-row cost before the clip and the clipped deltas scaled by w."""
    prestates, actions, rewards, poststates, terminals = minibatch
    w = np.asarray(w, F32)
    postq = O.forward(net.target_weights, poststates)
    maxpostq = postq.max(axis=1)
    preq, acts = O.forward(net.weights, prestates, keep=True)
    targets = O.td_targets(preq, maxpostq, actions, rewards, terminals, net.discount_rate, net.min_reward,
                           net.max_reward)
    deltas = preq - targets
    td = deltas[np.arange(len(actions)), actions].copy()
    cost = F32(np.mean(w * (np.sum(np.square(deltas), axis=1) / F32(2.0))))
    if net.clip_error:
        deltas = np.clip(deltas, -net.clip_error, net.clip_error)
    deltas = (deltas * w[:, None]).astype(F32)
    grads = O.backward(net.weights, acts, deltas)
    assert net.optimizer == "rmsprop"
    O.rmsprop_update(net.weights, net.states, grads, prestates.shape[0], net.learning_rate, net.decay_rate)
    net.train_iterations += 1
    net.last = dict(preq=preq, postq=postq, targets=targets, deltas=deltas, grads=grads, cost=cost, td=td)
    return cost
