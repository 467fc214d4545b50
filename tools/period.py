"""Developer tool: steady-state period (us per fused train step) of the production graph, device-timed, no tracing."""
import os, sys, random
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bench import make_args, synthetic_meta, NUM_ACTIONS
from simple_dqn_b200 import DeepQNetwork, ReplayMemory
st = torch.cuda.Stream()
torch.cuda.set_stream(st)
replay = 50000
base, actions, rewards, terminals = synthetic_meta(replay)
B = int(os.environ.get("BATCH", "32"))
HIST = int(os.environ.get("HIST", "4"))   # --history_length: frames per state, conv1's input channels
DOUBLE = os.environ.get("DOUBLE", "0") == "1"   # the Double DQN target (a third forward slot)
PER = os.environ.get("PER", "0") == "1"         # prioritized replay (tree-descent sampler + priority update)
NSTEP = int(os.environ.get("NSTEP", "1"))       # n-step returns (poststates N frames on, discounted reward sum)
ATOMS = int(os.environ.get("ATOMS", "0"))       # distributional head (C51) with this many atoms; 0: the scalar head
NACT = int(os.environ.get("NACT", str(NUM_ACTIONS)))   # actions (the replayed actions stay below 4)
DUELING = os.environ.get("DUELING", "0") == "1"   # dueling network (1024-unit fc1, advantage and value streams)
QUANTILES = int(os.environ.get("QUANTILES", "0"))   # quantile-regression head (QR-DQN) with this many quantiles; 0: off
MUNCHAUSEN = os.environ.get("MUNCHAUSEN", "0") == "1"   # the Munchausen target (extra target pass on the prestates)
IQN = int(os.environ.get("IQN", "0"))   # IQN head with this many tau samples per train row; 0: off
IQN_K = int(os.environ.get("IQN_K", "32"))   # the IQN head's tau samples per predict row
SHIFT = int(os.environ.get("SHIFT", "0"))   # random-shift augmentation with this pad p (DrQ: 4); 0: off
REM = int(os.environ.get("REM", "0"))   # random ensemble mixture head (REM) with this many heads per action; 0: off
FQF = int(os.environ.get("FQF", "0"))   # FQF head with this many fractions per sample; 0: off
BOOT = int(os.environ.get("BOOT", "0"))   # bootstrapped DQN heads, this many per action; 0: off
BOOT_P = float(os.environ.get("BOOT_P", "0.5"))   # the bootstrapped heads' mask probability
TAU = float(os.environ.get("TAU", "0"))   # soft target update: blend the target towards the online net by TAU every step
MAX_GRAD_NORM = float(os.environ.get("MAX_GRAD_NORM", "0"))   # global gradient-norm clipping at this norm; 0: off


def args():
    a = make_args(B)
    a.history_length = HIST
    a.double_dqn = DOUBLE
    a.prioritized_replay = PER
    a.n_step = NSTEP
    a.distributional = ATOMS > 0
    a.num_atoms = ATOMS
    a.dueling = DUELING
    a.quantile_regression, a.num_quantiles = QUANTILES > 0, QUANTILES
    a.munchausen = MUNCHAUSEN
    a.implicit_quantiles, a.num_tau_samples, a.num_quantile_samples = IQN > 0, IQN, IQN_K
    a.random_shift = SHIFT
    a.rem, a.num_heads = REM > 0, REM
    a.fqf, a.num_fractions = FQF > 0, FQF
    a.bootstrapped, a.bootstrap_heads, a.bootstrap_p = BOOT > 0, BOOT, BOOT_P
    a.soft_target_tau = TAU
    a.max_grad_norm = MAX_GRAD_NORM
    return a


mem = ReplayMemory(replay, args(), stream=st, rng="device")
for s in range(0, replay, 10000):
    mem.add_batch(actions[s:s + 10000], rewards[s:s + 10000], base, terminals[s:s + 10000])
mem.set_cursor(replay, 1234)
net = DeepQNetwork(NACT, args(), stream=st, math_mode=os.environ.get("MATH", "tcgen05"))
net.update_target_network()
random.seed(1); mem.seed_device_rng(random)
net.train_fused(mem, 300); st.synchronize()
ts = st
res = []
for rep in range(int(os.environ.get("REPS", "5"))):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(ts)
    net.train_fused(mem, 2000)
    e1.record(ts)
    st.synchronize()
    res.append(e0.elapsed_time(e1) / 2000 * 1e3)
import time
for _ in range(2):
    st.synchronize()
    t = time.time(); net.train_fused(mem, 300); t_enq = time.time() - t; st.synchronize(); t_all = time.time() - t
    print("300 steps: host enqueue %.1f us/step, until done %.1f us/step" % (t_enq / 300 * 1e6, t_all / 300 * 1e6))
print("math %s batch %d hist %d double %d per %d nstep %d actions %d atoms %d dueling %d quantiles %d munchausen %d iqn %d shift %d rem %d fqf %d boot %d boot_p %g tau %g max_grad_norm %g period_us min %.2f median %.2f  "
      "all %s" % (net.math_mode, B, HIST, DOUBLE, PER, NSTEP, NACT, ATOMS, DUELING, QUANTILES, MUNCHAUSEN, IQN, SHIFT, REM, FQF, BOOT, BOOT_P, TAU, MAX_GRAD_NORM, min(res), float(np.median(res)),
                  " ".join("%.2f" % r for r in res)))
