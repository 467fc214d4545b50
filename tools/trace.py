"""Developer tool: print the in-kernel timeline of one tensor-core kernel (B200DQN_TRACE_LABEL=conv23_fwd ...)."""
import os, sys, types
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from simple_dqn_b200 import DeepQNetwork, _lib as L
from bench import make_args
label = os.environ.get("B200DQN_TRACE_LABEL", "conv23_fwd")
net = DeepQNetwork(4, make_args(32), math_mode="tcgen05")
mb = (np.random.randint(0, 256, (32, 4, 84, 84)).astype(np.uint8), np.zeros(32, np.uint8), np.zeros(32, np.int64),
      np.random.randint(0, 256, (32, 4, 84, 84)).astype(np.uint8), np.zeros(32, np.uint8))
for _ in range(3):
    net.train(mb, 0)
t = L.debug_trace().astype(np.int64)
t0 = t[0]
# conv23_fwd: slots 3/4 close its conv2 phase, 2 marks H2 in shared memory, 7 its conv3 accumulators, k-blocks 8.. are conv3's
names = {0: "start", 1: "alloc+init done", 3: "loader0: all loads issued", 4: "accumulators ready",
         2: "conv23: H2 in shared memory", 7: "conv23: conv3 accumulators ready", 5: "epilogue stores done", 6: "end"}
for k in (0, 1, 3, 4, 2, 7, 5, 6):
    if t[k]:
        print("%-34s %8d" % (names[k], t[k] - t0))
print("kblk: mma_ready  mma_issued | ld0_stage_free  ld0_issued   (cycles since start)")
for it in range((len(t) - 8) // 4):
    row = t[8 + it * 4: 8 + it * 4 + 4]
    if not row.any(): break
    print(it, " ".join("%8d" % (x - t0 if x else -1) for x in row))
