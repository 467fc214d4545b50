"""Developer tool: GPU timeline of ONE steady-state fused train step inside the replayed CUDA graph (all branches, PDL)."""
import os, sys, random
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import make_args, synthetic_meta, NUM_ACTIONS
from simple_dqn_b200 import DeepQNetwork, ReplayMemory, Stream, _lib as L
st = Stream()
replay = 50000
base, actions, rewards, terminals = synthetic_meta(replay)
B = int(os.environ.get("BATCH", "32"))
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


def net_args():
    a = make_args(B)
    a.distributional, a.num_atoms = ATOMS > 0, ATOMS
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


mem = ReplayMemory(replay, make_args(B), stream=st, rng="device")
for s in range(0, replay, 10000):
    mem.add_batch(actions[s:s + 10000], rewards[s:s + 10000], base, terminals[s:s + 10000])
mem.set_cursor(replay, 1234)
net = DeepQNetwork(NACT, net_args(), stream=st, math_mode=os.environ.get("MATH", "tcgen05"))
net.update_target_network()
random.seed(1); mem.seed_device_rng(random)
net.train_fused(mem, 50); st.synchronize()
L.ktrace_begin(0, step=12)
net.train_fused(mem, 16); st.synchronize()     # re-captures with timing slots, records the 12th step of the batch
rows = L.ktrace_end()
t0 = min(r[1] for r in rows)
print("%-14s %9s %9s %8s" % ("kernel", "start_us", "end_us", "dur_us"))
for name, a, b in sorted(rows, key=lambda r: r[1]):
    print("%-14s %9.2f %9.2f %8.2f" % (name, (a - t0) / 1e3, (b - t0) / 1e3, (b - a) / 1e3))
print("step span %.2f us" % ((max(r[2] for r in rows) - t0) / 1e3))
