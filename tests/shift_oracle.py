"""Random-shift augmentation (DrQ, Kostrikov, Yarats and Fergus, 2020) on the CPU: a numpy restatement of the device's
k_shift_draw and of the shifted gather of conv1's kernels (csrc/net.cu, net_simt.cuh, net_umma.cu).  p = random_shift,
b the sample, z the slot (0 the prestates, 1 the poststates).

Rules (include/b200dqn.h states them too):
  1. x = mix(mix(seed + 0x9E3779B97F4A7C15 (ctr + 1)) ^ (z << 32 | b)), mix = splitmix64's finaliser, all mod 2^64;
     dy = ((x >> 32) (2p + 1) >> 32) - p and dx = ((x & 0xffffffff) (2p + 1) >> 32) - p.
  2. The shifted state's pixel (f, y, x) is frame f's pixel (clip(y + dy, 0, 83), clip(x + dx, 0, 83)), one (dy, dx)
     for every frame of the state: edge-replicate padding by p, then the 84x84 crop at (p + dy, p + dx).
  3. Slot 0's offsets shift the prestates (the online network and the Munchausen target pass), slot 1's the poststates
     (the target network and Double DQN's online network on the poststates).
"""
import numpy as np

U64 = np.uint64
SIDE = 84


def mix(x):
    """splitmix64's finaliser on uint64 arrays (numpy's uint64 arithmetic wraps mod 2^64)."""
    x = np.asarray(x, dtype=U64)
    with np.errstate(over="ignore"):
        x = x ^ (x >> U64(30))
        x = x * U64(0xBF58476D1CE4E5B9)
        x = x ^ (x >> U64(27))
        x = x * U64(0x94D049BB133111EB)
        x = x ^ (x >> U64(31))
    return x


def draw(seed, ctr, pad, batch):
    """Rule 1: the (2, batch, 2) int32 offsets (dy, dx) a train step draws at counter value `ctr`."""
    with np.errstate(over="ignore"):
        base = mix(U64(seed) + U64(0x9E3779B97F4A7C15) * (U64(ctr) + U64(1)))
    z = np.arange(2, dtype=U64)[:, None]
    b = np.arange(batch, dtype=U64)[None, :]
    x = mix(base ^ ((z << U64(32)) | b))
    span = U64(2 * pad + 1)
    dy = ((x >> U64(32)) * span) >> U64(32)
    dx = ((x & U64(0xFFFFFFFF)) * span) >> U64(32)
    return np.stack([dy.astype(np.int64) - pad, dx.astype(np.int64) - pad], axis=-1).astype(np.int32)


def shift(states, offsets):
    """Rule 2 on (n, H, 84, 84) uint8 states with (n, 2) offsets: the clamp form, as the kernels address it."""
    states = np.asarray(states)
    out = np.empty_like(states)
    r = np.arange(SIDE)
    for i, (dy, dx) in enumerate(np.asarray(offsets)):
        ys = np.clip(r + dy, 0, SIDE - 1)
        xs = np.clip(r + dx, 0, SIDE - 1)
        out[i] = states[i][:, ys][:, :, xs]
    return out


def shift_padded(states, offsets, pad):
    """Rule 2 in DrQ's own words: np.pad by `pad` with the edge values, then the crop at (pad + dy, pad + dx)."""
    states = np.asarray(states)
    out = np.empty_like(states)
    for i, (dy, dx) in enumerate(np.asarray(offsets)):
        padded = np.pad(states[i], ((0, 0), (pad, pad), (pad, pad)), mode="edge")
        out[i] = padded[:, pad + dy:pad + dy + SIDE, pad + dx:pad + dx + SIDE]
    return out


def shift_minibatch(minibatch, offsets):
    """Rule 3: a (pre, actions, rewards, post, terminals) host tuple as the network sees it under (2, batch, 2)
    offsets."""
    pre, act, rew, post, term = minibatch
    return shift(pre, offsets[0]), act, rew, shift(post, offsets[1]), term
