"""Every GEMM-shaped kernel against its float64 reference (tests/kernel_ref.py), fed the device's own inputs.

Each kernel's output is compared with the f64 layer applied to what the device itself fed that kernel: its H1..H4,
its dZ4..dZ1 and the pre-update weights.  So an error does not carry over from one layer to the next and no Rectlin
mask can flip.  The bound is elementwise and scaled by the operands (kernel_ref's docstring); a dropped lo term, a
skipped k-block or a wrong tile tail exceeds it, and tests/test_kernel_ref.py shows that on the CPU.

The head is restated bit for bit: the deltas from the device's preq/postq, dZ4 = δ·W5 under the H4 mask.

The test_double_* cases run the same checks on Double DQN steps, where every forward launch carries a third network
slot (the online net on the poststates) and the deltas and cost follow the Double DQN target (head_restated).

Batch sweep of the tensor-core engine (A = 4, H = 4) and what each size runs (kernel_ref.dispatch):

    batch                 1    2    3   16   33   63   64   65  128  129  256  257  512  4096 (forward only)
    conv2/conv3 forward   conv23_fwd (one kernel) ------------>   conv2_fwd + conv3_fwd ------------------->
    fc1_fwd splits        7 ---------------------------------------------------------->   4 ------------->
    conv1_wgrad splits    1    2    3   13   26   44   45   46   48   48   48   48   48
    conv2_wgrad splits    1    1    1    6   11   20   21   21   41   41   47   47   47
    conv3_wgrad splits    1    1    1    4    7   13   13   13   25   25   40   40   44
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import kernel_ref as K
from double_oracle import head_restated
from helpers import make_args, rel_l2

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SWEEP = [1, 2, 3, 16, 33, 63, 64, 65, 128, 129, 256, 257, 512]
SCHEDS = ["serial", "branches"]
F32 = np.float32
WORST = {}          # kernel -> largest ratio of error to bound seen in this module (vanilla steps and predicts)
WORST_DOUBLE = {}   # the same for the Double DQN steps


def _note(ratios, double=False):
    worst = WORST_DOUBLE if double else WORST
    for k, v in ratios.items():
        worst[k] = max(worst.get(k, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nlargest |error| / bound per kernel:  vanilla   double")
    for k in sorted(set(WORST) | set(WORST_DOUBLE)):
        print("  %-20s %11s %8s" % (k, *("%.3g" % w[k] if k in w else "-" for w in (WORST, WORST_DOUBLE))))


def minibatch(n, hist, num_actions, seed, terminal_p=0.3, rewards=(-3, 4), states=None):
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8) if states is None else states
    post = rs.randint(0, 256, (n, hist, 84, 84)).astype(np.uint8) if states is None else states.copy()
    return (pre, rs.randint(0, num_actions, n).astype(np.uint8),
            rs.randint(rewards[0], rewards[1], n).astype(np.int64), post, rs.rand(n) < terminal_p)


def make_net(batch, engine="tcgen05", hist=4, num_actions=4, sched="branches", seed=3, w5_scale=3.0, keep=True,
             double=False, **kw):
    """A net with Xavier weights, fc1 × 3 and fc2 × w5_scale (Q of order 1, like a trained net), small RMSProp
    state and a freshly synced target.  double: the Double DQN target, with target weights perturbed away from the
    online ones (by 0.3·max|W| of noise per layer), so that the two networks prefer different poststate actions."""
    from simple_dqn_b200 import DeepQNetwork, Stream
    net = DeepQNetwork(num_actions, make_args(batch_size=batch, history_length=hist, random_seed=seed,
                                              double_dqn=double, **kw),
                       math_mode=engine, stream=Stream() if sched == "branches" else None)
    ws, _ = net.get_weights()
    ws[3] = ws[3] * F32(3.0)
    ws[4] = ws[4] * F32(w5_scale)
    rs = np.random.RandomState(seed)
    net.set_weights(ws, [np.abs(rs.randn(*w.shape)).astype(F32) * F32(1e-4) for w in ws])
    net.update_target_network()
    if double:
        net.set_weights([(w + rs.randn(*w.shape).astype(F32) * F32(0.3) * np.abs(w).max()).astype(F32) for w in ws],
                        None, which=1)
    net.keep_grads(keep)
    return net


def _chain(engine, kernel, rows, hist, fc1_forced=0, hidden=K.HIDDEN):
    """hidden: fc1's width (512, or 1024 on a dueling net), the reduction length of fc1_dgrad."""
    if engine == "tcgen05":
        return K.chain(kernel, rows, hist, fc1_forced, hidden)
    full = {"conv1_fwd": 64 * hist, "conv2_fwd": 512, "conv3_fwd": 576, "fc1_fwd": K.FLAT, "fc1_dgrad": hidden,
            "conv3_dgrad": 576, "conv2_dgrad": 1024, "fc1_wgrad": rows, "conv3_wgrad": rows * 49,
            "conv2_wgrad": rows * 81, "conv1_wgrad": rows * 400}
    return full[kernel]


def _check(name, engine, op, a, b, dev, n, mask=None, post=None, a_exact=False, split=None):
    """ratio of |dev - f64 reference| to the bound; mask: Rectlin mask of the output, post: Rectlin on the output"""
    y = op(a, b)
    bnd = K.bound(op, a, b, n, y, split=(engine == "tcgen05") if split is None else split, a_exact=a_exact)
    if mask is not None:
        y, bnd = y * mask, bnd * mask
    if post is not None:
        y = post(y)
    return {name: K.ratio(dev, y, bnd)}


def gemm_forward_ratios(engine, states, ws, acts, fc1_forced=0):
    """conv1..conv3 and fc1 forward, each against its f64 layer on the device's own inputs; fc1 at its width
    (ws[3]'s rows)."""
    rows, hist = states.shape[0], states.shape[1]
    h1, h2, h3, h4 = acts
    r = {}
    for name, op, a, b, dev, exact in (("conv1_fwd", K.conv_fwd(0), K.states_f64(states), ws[0], h1, True),
                                       ("conv2_fwd", K.conv_fwd(1), h1, ws[1], h2, False),
                                       ("conv3_fwd", K.conv_fwd(2), h2, ws[2], h3, False),
                                       ("fc1_fwd", K.fc_fwd, h3, ws[3], h4, False)):
        r.update(_check(name, engine, op, a, b, dev, _chain(engine, name, rows, hist, fc1_forced), post=K.relu,
                        a_exact=exact))
    return r


def forward_ratios(engine, states, ws, acts, q, fc1_forced=0):
    r = gemm_forward_ratios(engine, states, ws, acts, fc1_forced)
    r.update(_check("fc2_fwd", engine, K.fc_fwd, acts[3], ws[4], q, K.HIDDEN, split=False))   # the head: CUDA cores
    return r


def gemm_backward_ratios(engine, states, ws, acts, dz, grads):
    """The seven GEMM-shaped backward kernels (fc1 and conv dgrads and wgrads), each against its f64 layer on the
    device's own dZ and activations; fc1_dgrad reduces over fc1's width (ws[3]'s rows)."""
    rows, hist = states.shape[0], states.shape[1]
    h1, h2, h3, h4 = acts
    dz1, dz2, dz3, dz4 = dz
    c = lambda k: _chain(engine, k, rows, hist, hidden=ws[3].shape[0])
    fc1_dgrad = lambda a, b: K.fc_dgrad(a, b).reshape(len(a), 64, 7, 7)
    r = {}
    r.update(_check("fc1_dgrad", engine, fc1_dgrad, dz4, ws[3], dz3, c("fc1_dgrad"), mask=h3 > 0))
    r.update(_check("conv3_dgrad", engine, K.conv_dgrad(2), dz3, ws[2], dz2, c("conv3_dgrad"), mask=h2 > 0))
    r.update(_check("conv2_dgrad", engine, K.conv_dgrad(1), dz2, ws[1], dz1, c("conv2_dgrad"), mask=h1 > 0))
    r.update(_check("fc1_wgrad", engine, K.fc_wgrad, h3, dz4, grads[3], c("fc1_wgrad")))
    r.update(_check("conv3_wgrad", engine, K.conv_wgrad(2), h2, dz3, grads[2], c("conv3_wgrad")))
    r.update(_check("conv2_wgrad", engine, K.conv_wgrad(1), h1, dz2, grads[1], c("conv2_wgrad")))
    r.update(_check("conv1_wgrad", engine, K.conv_wgrad(0), K.states_f64(states), dz1, grads[0], c("conv1_wgrad"),
                    a_exact=True))
    return r


def backward_ratios(engine, states, ws, acts, dz, grads, deltas):
    # dZ4 = δ·W5 under the H4 mask: one fp32 product per element (k_head / the SIMT head alike)
    h4, dz4 = acts[3], dz[3]
    ref4 = (deltas.astype(F32) @ ws[4]) * (h4 > 0)
    assert (dz4 == ref4).all(), np.abs(dz4 - ref4).max()
    r = gemm_backward_ratios(engine, states, ws, acts, dz, grads)
    r.update(_check("fc2_wgrad", engine, K.fc_wgrad, h4, deltas, grads[4], len(states), split=False))
    return r


def train_and_check(net, mb, fc1_forced=0, clip=1.0, min_reward=-1, max_reward=1):
    """One train step, every kernel of it held to its bound; then predict on fresh states with the updated weights
    (the refreshed tile images, lo halves included).  Returns the ratios and the train step's device tensors."""
    engine = net.math_mode
    ws0 = net.get_weights(with_states=False)
    net.train(mb, 0)
    pre = mb[0]
    preq, postq = net.last_q()
    acts = net.last_activations()
    if net.double_dqn:      # the target values the action the online network picks on the poststates
        oq = net.last_online_postq()
        raw, clipped = (head_restated(preq, postq, oq, mb[1], mb[2], mb[4], min_reward=min_reward,
                                      max_reward=max_reward, clip=c)[0] for c in (0, clip))
    else:
        raw, clipped = K.head_td(preq, postq, mb[1], mb[2], mb[4], clip=clip, min_reward=min_reward,
                                 max_reward=max_reward)
    deltas = net.last_deltas()
    assert (deltas == clipped).all(), np.abs(deltas - clipped).max()
    row_cost = (F32(0.5) * raw * raw).sum(axis=1)          # one non-zero delta per row
    assert (net.last_row_costs() == row_cost).all()
    tot = F32(0)
    for c in row_cost:                                      # k_cost_finish: fp32, row order, then / rows
        tot = F32(tot + c)
    assert net.last_costs(1)[0] == F32(tot / F32(len(row_cost))), (net.last_costs(1)[0], tot)
    r = forward_ratios(engine, pre, ws0, acts, preq, fc1_forced)
    step = dict(acts=acts, dz=net.last_dz(), grads=net.get_grads())
    r.update(backward_ratios(engine, pre, ws0, acts, step["dz"], step["grads"], deltas))
    ws1 = net.get_weights(with_states=False)
    fresh = minibatch(len(pre), pre.shape[1], net.num_actions, 1234)[0]
    q = net.predict(fresh)
    r.update({k + "@updated": v for k, v in
              forward_ratios(engine, fresh, ws1, net.last_activations(), q, fc1_forced).items()})
    _note(r, net.double_dqn)
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, bad
    return r, step


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("batch", SWEEP)
def test_train_step_kernels(batch, sched):
    net = make_net(batch, sched=sched)
    train_and_check(net, minibatch(batch, 4, 4, 2))


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("batch", SWEEP)
def test_double_train_step_kernels(batch, sched):
    """Double DQN: every forward launch runs a third network slot (the online net on the poststates)."""
    net = make_net(batch, sched=sched, double=True)
    mb = minibatch(batch, 4, 4, 2)
    train_and_check(net, mb)
    if batch >= 33:         # the two networks disagree on some poststates: the Double DQN target is really in play
        assert (net.last_online_postq().argmax(1) != net.last_q()[1].argmax(1))[~mb[4]].any()


def test_forward_kernels_at_4096():
    net = make_net(4096)
    states = minibatch(4096, 4, 4, 5)[0]
    q = net.predict(states)
    _note(forward_ratios("tcgen05", states, net.get_weights(with_states=False), net.last_activations(), q))
    assert all(v <= 1.0 for v in WORST.values())


@pytest.mark.parametrize("hist", [1, 5, 16])
@pytest.mark.parametrize("batch", [1, 64, 65])
def test_history_lengths(hist, batch):
    net = make_net(batch, hist=hist)
    train_and_check(net, minibatch(batch, hist, 4, 3))


@pytest.mark.parametrize("hist", [1, 5, 16])
@pytest.mark.parametrize("batch", [1, 64, 65])
def test_double_history_lengths(hist, batch):
    net = make_net(batch, hist=hist, double=True)
    train_and_check(net, minibatch(batch, hist, 4, 3))


HEAD_CASES = {
    "A18": dict(num_actions=18),
    "A32": dict(num_actions=32),
    "rewards_asym": dict(min_reward=-2, max_reward=3, rewards=(-6, 7)),
    "all_terminal": dict(terminal_p=1.1),
    "no_terminal": dict(terminal_p=-0.1),
    "clip0": dict(clip_error=0, rewards=(-6, 7)),
}


@pytest.mark.parametrize("case", sorted(HEAD_CASES))
def test_head(case):
    kw = dict(HEAD_CASES[case])
    a = kw.pop("num_actions", 4)
    rewards, tp = kw.pop("rewards", (-3, 4)), kw.pop("terminal_p", 0.3)
    net = make_net(33, num_actions=a, **kw)
    mb = minibatch(33, 4, a, 7, terminal_p=tp, rewards=rewards)
    clip = float(kw.get("clip_error", 1))
    train_and_check(net, mb, clip=clip, min_reward=kw.get("min_reward", -1), max_reward=kw.get("max_reward", 1))
    d = np.abs(net.last_deltas()).max(axis=1)
    if clip:
        assert (d == clip).any() and ((d > 0) & (d < clip)).any()    # deltas on both sides of the clip
    else:
        assert d.max() > 1.0                                         # nothing was clipped


@pytest.mark.parametrize("value", [0, 255])
def test_constant_frames(value):
    net = make_net(33)
    states = np.full((33, 4, 84, 84), value, np.uint8)
    mb = minibatch(33, 4, 4, 9, states=states)
    train_and_check(net, mb)
    if value == 0:          # every Rectlin is off: Q = 0 and every gradient is exactly 0
        assert not any(g.any() for g in net.get_grads())
        assert not net.predict(states).any()
        assert not any(h.any() for h in net.last_activations())


SCALES = [1e-3, 1e-5, 1e-7]
REL = {}


@pytest.mark.parametrize("scale", SCALES)
def test_small_gradients(scale):
    """δ shrunk by shrinking W5, with zero rewards on terminal transitions (target 0, δ = Q).  The 2⁻³⁶ floor of the
    bound is what covers the lo planes falling into fp16 subnormals here; rel-L2 per weight gradient is printed."""
    from oracle import dqn_oracle as O
    mb = minibatch(32, 4, 4, 11, terminal_p=1.1, rewards=(0, 1))
    probe = make_net(32)
    ws = probe.get_weights(with_states=False)
    q = O.forward(ws, mb[0])
    w5_scale = 3.0 * scale / np.abs(q[np.arange(32), mb[1]]).max()
    net = make_net(32, w5_scale=w5_scale)
    r, step = train_and_check(net, mb)
    dmax = float(np.abs(net.last_deltas()).max())
    assert 0.3 * scale <= dmax <= 3 * scale, dmax
    # rel-L2 of each weight gradient against the f64 wgrad of the device's own operands
    states, acts, (dz1, dz2, dz3, dz4), grads = mb[0], step["acts"], step["dz"], step["grads"]
    refs = [K.conv_wgrad(0)(K.states_f64(states), dz1), K.conv_wgrad(1)(acts[0], dz2),
            K.conv_wgrad(2)(acts[1], dz3), K.fc_wgrad(acts[2], dz4)]
    REL[scale] = [rel_l2(g, ref) for g, ref in zip(grads, refs)]
    print("max|delta| %.2g: rel-L2 conv1..fc1 wgrad %s; worst ratio %.3g" %
          (dmax, " ".join("%.2g" % v for v in REL[scale]), max(r.values())))


@pytest.mark.parametrize("batch", [1, 33, 65, 256])
def test_target_net_equals_online_net(batch):
    """Freshly synced target, poststates = prestates: the target forward (the same kernels on blockIdx.z = 1, tile
    images copied at the sync) gives postq == preq bit for bit."""
    net = make_net(batch)
    net.train(minibatch(batch, 4, 4, 13), 0)      # the online images now differ from the ones the sync copied
    net.update_target_network()
    states = minibatch(batch, 4, 4, 14)[0]
    net.train(minibatch(batch, 4, 4, 15, states=states), 0)
    preq, postq = net.last_q()
    assert (preq == postq).all()


@pytest.mark.parametrize("sched", SCHEDS)
@pytest.mark.parametrize("batch", [32, 65])
def test_keep_grads_changes_nothing(sched, batch):
    nets = [make_net(batch, sched=sched, keep=k) for k in (False, True)]
    mb = minibatch(batch, 4, 4, 17)
    for net in nets:
        net.train(mb, 0)
    (g0, g1), (w0, w1) = [n.get_grads() for n in nets], [n.get_weights() for n in nets]
    assert all((a == b).all() for a, b in zip(g0, g1))
    assert all((a == b).all() for a, b in zip(w0[0] + w0[1], w1[0] + w1[1]))


@pytest.mark.parametrize("batch", [1, 32, 65])
def test_simt_engine_kernels(batch):
    net = make_net(batch, engine="fp32", sched="serial")
    train_and_check(net, minibatch(batch, 4, 4, 19))


@pytest.mark.parametrize("batch", [1, 32, 65])
def test_double_simt_engine_kernels(batch):
    net = make_net(batch, engine="fp32", sched="serial", double=True)
    train_and_check(net, minibatch(batch, 4, 4, 19))


def _child(env, cases, double=False):
    """Run train_and_check in a child process: the B200DQN_* switches are read once per process."""
    code = ("import json, sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "import test_gpu_kernels as T\n"
            "out = []\n"
            "for batch, kw in %r:\n"
            "    out.append(T.train_and_check(T.make_net(batch, double=%r), T.minibatch(batch, 4, 4, 21), **kw)[0])\n"
            "print('RATIOS', json.dumps(out))\n" % (ROOT, os.path.join(ROOT, "tests"), cases, double))
    out = subprocess.run([sys.executable, "-s", "-c", code], env=dict(os.environ, **env), capture_output=True,
                         text=True, timeout=900)
    assert out.returncode == 0, out.stderr[-4000:]
    line = [l for l in out.stdout.splitlines() if l.startswith("RATIOS ")][0]
    for r in json.loads(line[len("RATIOS "):]):
        _note(r, double)


@pytest.mark.parametrize("splits", [1, 4, 14])
def test_fc1_forced_splits(splits):
    _child({"B200DQN_FC1_SPLITS": str(splits)}, [(b, {"fc1_forced": splits}) for b in (33, 257)])


@pytest.mark.parametrize("splits", [1, 4, 14])
def test_double_fc1_forced_splits(splits):
    """Three slots of split-K partials: 14 forced splits fill the whole partial buffer."""
    _child({"B200DQN_FC1_SPLITS": str(splits)}, [(b, {"fc1_forced": splits}) for b in (33, 257)], double=True)
