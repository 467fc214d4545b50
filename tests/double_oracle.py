"""Double DQN train step (van Hasselt et al., 2016) on the CPU: the numpy oracle of oracle/dqn_oracle.py with the
poststate action chosen by the online network and valued by the target network.

    a*_i = argmax_a Q_online(s'_i, a)          (first index of the maximum, np.argmax)
    y_i  = r_i                                 if terminal_i
           r_i + discount * Q_target(s'_i, a*_i)  otherwise

The target is formed in Python floats (double) and stored into float32, as td_targets does for the max.  Everything
else (reward clip, cost before the delta clip, backward, optimizers) is the vanilla step's.  With double_dqn=False
the class is DQNOracle.
"""
import numpy as np

from oracle import dqn_oracle as O

F32 = np.float32


class DoubleDQNOracle(O.DQNOracle):
    def __init__(self, num_actions, double_dqn=False, **kw):
        super().__init__(num_actions, **kw)
        self.double_dqn = double_dqn
        self.pick = None    # optional online_postq -> a* (a test resolving near-ties the way the device did)

    def train(self, minibatch, epoch=0):
        if not self.double_dqn:
            return super().train(minibatch, epoch)
        prestates, actions, rewards, poststates, terminals = minibatch
        assert prestates.shape == poststates.shape and prestates.ndim == 4
        postq = O.forward(self.target_weights, poststates)
        online_postq = O.forward(self.weights, poststates)
        astar = self.pick(online_postq) if self.pick else np.argmax(online_postq, axis=1)
        chosen = postq[np.arange(len(astar)), astar]
        preq, acts = O.forward(self.weights, prestates, keep=True)
        targets = O.td_targets(preq, chosen, actions, rewards, terminals,
                               self.discount_rate, self.min_reward, self.max_reward)
        deltas = preq - targets
        cost = F32(np.mean(np.sum(np.square(deltas), axis=1) / F32(2.0)))
        if self.clip_error:
            deltas = np.clip(deltas, -self.clip_error, self.clip_error)
        grads = O.backward(self.weights, acts, deltas.astype(F32))
        if self.optimizer == "rmsprop":
            O.rmsprop_update(self.weights, self.states, grads, prestates.shape[0], self.learning_rate, self.decay_rate)
        elif self.optimizer == "adam":
            O.adam_update(self.weights, self.states, grads, prestates.shape[0], self.train_iterations + 1,
                          self.learning_rate)
        else:
            O.adadelta_update(self.weights, self.states, grads, prestates.shape[0], self.decay_rate)
        self.train_iterations += 1
        self.last = dict(preq=preq, postq=postq, online_postq=online_postq, astar=astar, targets=targets,
                         deltas=deltas, grads=grads, cost=cost)
        if self.callback:
            self.callback.on_train(cost)
        return cost


def head_restated(preq, postq, online_postq, actions, rewards, terminals, discount=0.99, min_reward=-1, max_reward=1,
                  clip=1.0):
    """The head's TD step on given fp32 Q rows, bit for bit: deltas (clipped), per-sample cost (before the clip)."""
    r = np.clip(rewards, min_reward, max_reward)
    n, A = preq.shape
    deltas = np.zeros((n, A), F32)
    row_cost = np.zeros(n, F32)
    for i in range(n):
        best = 0
        for j in range(1, A):                       # first index of the maximum
            if online_postq[i, j] > online_postq[i, best]:
                best = j
        y = float(r[i]) if terminals[i] else float(r[i]) + discount * float(postq[i, best])
        d = F32(preq[i, actions[i]] - F32(y))
        row_cost[i] = F32(0.5) * d * d
        if clip > 0:
            d = F32(min(max(d, F32(-clip)), F32(clip)))
        deltas[i, actions[i]] = d
    return deltas, row_cost
