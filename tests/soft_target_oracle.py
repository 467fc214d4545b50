"""The soft (Polyak-averaged) target update of include/b200dqn.h (b200dqn_net_config::soft_target_tau), restated in
numpy float32 with one rounding per operation:

    c = float32(1 - tau)   (1 - tau in float64 from the Python float)
    t = float32(tau)
    target' = fl(fl(c * target) + fl(t * online))

Every layer of the target network (0-4, the IQN / FQF embedding, the FQF fraction layer) takes this rule once per
train step, online being the weights after that step's optimizer update; the optimizer states are not touched."""
import numpy as np

F32 = np.float32


def factors(tau):
    """(c, t) of the rule for a float64 tau."""
    return F32(1.0 - float(tau)), F32(float(tau))


def blend(target, online, tau):
    """target' of the rule, elementwise, float32 (each product and the sum rounded on its own: numpy float32 ops do not
    contract)."""
    c, t = factors(tau)
    target = np.asarray(target, dtype=F32)
    online = np.asarray(online, dtype=F32)
    return (c * target) + (t * online)


def blend_layers(targets, onlines, tau):
    """The rule over a list of layers."""
    return [blend(a, b, tau) for a, b in zip(targets, onlines)]
