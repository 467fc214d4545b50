"""Float64 reference of every GEMM-shaped layer of the Q-network, an emulation of the tensor-core engine's hi/lo
operand scheme, and the elementwise error bound tests/test_gpu_kernels.py holds each kernel to.

Layouts are the oracle's (oracle/dqn_oracle.py): activations NCHW, conv weights W[(c, r, s), k], linear weights
W[out, in].  Every layer function takes its inputs explicitly and returns float64, so a test can feed each kernel's
reference with the device's own inputs and no error carries over from one layer to the next.  Every reference
operation ``op(a, b)`` is bilinear in its two operands; the bound evaluates the same ``op`` on squared operands.

The scheme (DESIGN §4).  Every fp32 operand x is split into ``hi = fp16(x)`` and ``lo = fp16((x - hi)·2¹¹)``
(round to nearest even, subnormals kept) and a kernel computes ``A_hi·B_hi + (A_hi·B_lo + A_lo·B_hi)·2⁻¹¹`` with fp32
accumulators.  conv1's A operand (u8 pixels) is exact and has no lo plane.

Error model.  For one output y = Σ_k a_k·b_k:
  * each operand is represented to ≤ 2⁻²²·|x| + 2⁻³⁶ (the second term is half the subnormal spacing of lo, scaled
    back by 2⁻¹¹), and the dropped A_lo·B_lo term is ≤ 2⁻²²·|a·b|.  These errors change sign from term to term, so
    their sum grows like S₂ = sqrt(Σ a_k²·b_k²), not like Σ|a_k·b_k|;
  * fp32 accumulation over the kernel's longest serial chain of n additions (k-blocks per split × 64, plus the
    split-K reduction; :func:`chain`) adds random-signed roundings of the running sums, ≈ 2⁻²⁴·√n·S₂;
  * the epilogue rounds y to fp32 (conv1 also multiplies by fp32 1/255).
giving, elementwise,

    bound = C_REP·2⁻²²·S₂ + C_ACC·2⁻²⁴·√n·S₂ + C_OUT·2⁻²⁴·|y| + C_FLOOR·2⁻³⁶·(sqrt(Σ a_k²) + sqrt(Σ b_k²))

with C_REP = C_ACC = C_OUT = C_FLOOR = 16 (:data:`C`).  Where a Rectlin mask is off the bound is 0: the kernels
write an exact 0 there.  Rectlin itself is 1-Lipschitz, so a forward layer's bound is that of its pre-activation.
Plain fp32 kernels (the head's fc2, the SIMT engine) use the same formula without the representation and floor
terms, with n = the full reduction length.

Calibration (tests/test_kernel_ref.py, at every batch of the GPU sweep): the emulated scheme, with f64 sums and, for
the weight gradients, with fp32 accumulation in k-block and split-K order, stays at least 4× inside the bound.
A dropped A_lo or B_lo term, lo scaled by 2¹⁰, one skipped k-block, one dropped split-K partial, a zeroed last row
and a stale lo weight image each exceed it; so does, on the dueling net's 1024-wide fc1, one of its two 512-unit
streams dropped from fc1_fwd's output or from fc1_dgrad's reduction.  A dropped lo term costs ≈ 2⁻¹²·S₂ per output, about 2⁸ times the
C_REP term; the constants sit between the two with room on both sides.
"""
import numpy as np

F64 = np.float64
LO_SCALE = 2.0 ** 11
C = dict(rep=16.0, acc=16.0, out=16.0, floor=16.0)

CONV = [(8, 8, 32, 4), (4, 4, 64, 2), (3, 3, 64, 1)]      # (R, S, K, stride), deepqnetwork.py:83-87
HW = [84, 20, 9, 7]                                       # input side of conv1, conv2, conv3; conv3's output side
HIDDEN, FLAT = 512, 3136


# ---- float64 layers ---------------------------------------------------------------------------------------------
def im2col(x, layer):
    """x (N, C, H, W) -> (N·P·Q, C·R·S) in (c, r, s) column order, the rows of the Neon weight."""
    r, s, _, st = CONV[layer]
    n, c, h, w = x.shape
    p, q = (h - r) // st + 1, (w - s) // st + 1
    win = np.lib.stride_tricks.sliding_window_view(x, (r, s), axis=(2, 3))[:, :, ::st, ::st]
    return np.ascontiguousarray(win.transpose(0, 2, 3, 1, 4, 5)).reshape(n * p * q, c * r * s), p, q


def conv_fwd(layer):
    """Pre-activation of conv layer `layer` (0..2): (x NCHW, W[(c,r,s), k]) -> NCHW."""
    def op(x, w):
        cols, p, q = im2col(np.asarray(x, F64), layer)
        z = cols @ np.asarray(w, F64)
        return z.reshape(x.shape[0], p, q, -1).transpose(0, 3, 1, 2)
    return op


def conv_dgrad(layer):
    """Gradient at conv layer `layer`'s input (1..2) from dZ at its output: (dZ NCHW, W) -> NCHW, unmasked."""
    r, s, k, st = CONV[layer]
    hin = HW[layer]

    def op(dz, w):
        dz, w = np.asarray(dz, F64), np.asarray(w, F64)
        n, _, p, q = dz.shape
        c = w.shape[0] // (r * s)
        cols = (dz.transpose(0, 2, 3, 1).reshape(-1, k) @ w.T).reshape(n, p, q, c, r, s)
        dx = np.zeros((n, c, hin, hin))
        for rr in range(r):
            for ss in range(s):
                dx[:, :, rr:rr + st * p:st, ss:ss + st * q:st] += cols[:, :, :, :, rr, ss].transpose(0, 3, 1, 2)
        return dx
    return op


def conv_wgrad(layer):
    """Weight gradient of conv layer `layer`, summed over the batch: (x NCHW, dZ NCHW) -> W[(c,r,s), k]."""
    def op(x, dz):
        cols, _, _ = im2col(np.asarray(x, F64), layer)
        dz = np.asarray(dz, F64)
        return cols.T @ dz.transpose(0, 2, 3, 1).reshape(-1, dz.shape[1])
    return op


def fc_fwd(x, w):
    return np.asarray(x, F64).reshape(len(x), -1) @ np.asarray(w, F64).T


def fc_dgrad(dz, w):
    return np.asarray(dz, F64) @ np.asarray(w, F64)


def fc_wgrad(x, dz):
    return np.asarray(dz, F64).T @ np.asarray(x, F64).reshape(len(x), -1)


def relu(z):
    return np.maximum(z, 0.0)


def states_f64(states_u8):
    return np.asarray(states_u8, F64) / 255.0


# ---- dispatch of the tensor-core engine (net_umma.cu) ---------------------------------------------------------
def fc1_splits(rows, forced=0):
    """fc1_fwd's split-K count (fc1_splits_for)."""
    return forced if 1 <= forced <= 14 else (7 if rows <= 256 else 4)


def wgrad_split(layer, rows):
    """(k-blocks per split, splits) of conv layer `layer`'s weight gradient (umma_wgrad_kb / umma_wgrad_splits)."""
    kred = rows * (400, 81, 49)[layer]
    kbs = (kred + 63) // 64
    per = (kbs + 47) // 48
    if layer == 0:
        per = max(per, 8)
    per = max(per, 4)
    return per, (kbs + per - 1) // per


def chain(kernel, rows, hist=4, fc1_forced=0, hidden=HIDDEN):
    """Longest serial fp32 accumulation chain of one output of `kernel` at `rows` samples.  hidden: fc1's width (512,
    or 1024 on a dueling net), which fc1_dgrad reduces over."""
    fixed = {"conv1_fwd": 64 * hist, "conv2_fwd": 512, "conv3_fwd": 576, "fc1_dgrad": hidden, "conv3_dgrad": 576,
             "conv2_dgrad": 256}
    if kernel in fixed:
        return fixed[kernel]
    if kernel == "fc1_fwd":
        sp = fc1_splits(rows, fc1_forced)
        return -(-49 // sp) * 64 + sp
    if kernel == "fc1_wgrad":
        return -(-rows // 64) * 64
    layer = {"conv1_wgrad": 0, "conv2_wgrad": 1, "conv3_wgrad": 2}[kernel]
    per, sp = wgrad_split(layer, rows)
    return min(per * 64, rows * (400, 81, 49)[layer]) + sp


def dispatch(rows, hist=4, hidden=HIDDEN):
    """What the engine runs at `rows` samples, for test ids and reports."""
    return dict(conv23=rows <= 64, fc1_splits=fc1_splits(rows), fc1_width=hidden,
                wgrad_splits=tuple(wgrad_split(l, rows)[1] for l in range(3)))


# ---- the error bound --------------------------------------------------------------------------------------------
def bound(op, a, b, n, y=None, split=True, a_exact=False):
    """Elementwise bound on |kernel(a, b) - op(a, b)| (module docstring).  split=False: plain fp32 operands."""
    a, b = np.asarray(a, F64), np.asarray(b, F64)
    y = op(a, b) if y is None else y
    s2 = np.sqrt(op(a * a, b * b))
    out = (C["acc"] * 2.0 ** -24 * np.sqrt(n)) * s2 + C["out"] * 2.0 ** -24 * np.abs(y)
    if split:
        out += C["rep"] * 2.0 ** -22 * s2
        out += C["floor"] * 2.0 ** -36 * np.sqrt(op(a * a, np.ones_like(b)))
        if not a_exact:
            out += C["floor"] * 2.0 ** -36 * np.sqrt(op(np.ones_like(a), b * b))
    return out


def ratio(dev, ref, bnd):
    """max |dev - ref| / bnd; an element with bound 0 must match exactly."""
    err = np.abs(np.asarray(dev, F64) - ref)
    if (err[bnd == 0] > 0).any():
        return float("inf")
    live = bnd > 0
    return float((err[live] / bnd[live]).max()) if live.any() else 0.0


# ---- emulation of the scheme ------------------------------------------------------------------------------------
def split(x, scale=LO_SCALE):
    """(hi, lo) fp16 planes of fp32 x, as the kernels' epilogues write them (__float2half_rn)."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = ((x - hi.astype(np.float32)) * np.float32(scale)).astype(np.float16)
    return hi, lo


def gemm_hilo(op, a, b, a_exact=False, lo_scale=LO_SCALE, drop_a_lo=False, drop_b_lo=False, b_lo_from=None):
    """op(a, b) computed from fp16 planes as the tensor-core kernels do, with float64 sums.  b_lo_from: take B's lo
    plane from this (older) tensor instead (a stale lo image)."""
    ah, al = split(a, lo_scale)
    bh, bl = split(b, lo_scale)
    if b_lo_from is not None:
        bl = split(b_lo_from, lo_scale)[1]
    ah, al, bh, bl = (np.asarray(t, F64) for t in (ah, al, bh, bl))
    if a_exact:
        ah, drop_a_lo = np.asarray(a, F64), True
    out = op(ah, bh)
    cross = 0.0
    if not drop_b_lo:
        cross = cross + op(ah, bl)
    if not drop_a_lo:
        cross = cross + op(al, bh)
    return out + np.asarray(cross) / LO_SCALE


def planes_f64(x):
    hi, lo = split(x)
    return np.asarray(hi, F64), np.asarray(lo, F64)


def wgrad_fp32_chunked(x_cols, dz_rows, per, splits, a_exact=False):
    """Weight gradient x_colsᵀ·dz_rows from hi/lo planes, the reduction (rows = pixels or samples) run as the kernel
    does: each 64-row k-block summed exactly and added to an fp32 accumulator, k-blocks in order inside a split,
    then the split partials reduced in fp32 in k_opt_conv's order (eight strided running sums, then a pairwise
    tree)."""
    k = x_cols.shape[0]
    parts = []
    for sp in range(splits):
        acc = np.zeros((x_cols.shape[1], dz_rows.shape[1]), np.float32)
        for kb in range(sp * per, min((sp + 1) * per, -(-k // 64))):
            s = slice(kb * 64, (kb + 1) * 64)
            bh, bl = planes_f64(dz_rows[s])
            if a_exact:
                ah, al = np.asarray(x_cols[s], F64), 0.0 * np.asarray(x_cols[s], F64)
            else:
                ah, al = planes_f64(x_cols[s])
            blk = ah.T @ bh + (ah.T @ bl + al.T @ bh) / LO_SCALE
            acc = (acc + blk.astype(np.float32)).astype(np.float32)
        parts.append(acc)
    lanes = [np.zeros_like(parts[0]) for _ in range(8)]
    for sp, p in enumerate(parts):
        lanes[sp % 8] = (lanes[sp % 8] + p).astype(np.float32)
    o = 1
    while o < 8:
        for u in range(0, 8, 2 * o):
            lanes[u] = (lanes[u] + lanes[u + o]).astype(np.float32)
        o *= 2
    return lanes[0].astype(F64)


# ---- the head (net.cu::k_head), restated bit for bit --------------------------------------------------------------
def head_td(preq, postq, actions, rewards, terminals, discount=0.99, min_reward=-1, max_reward=1, clip=1.0):
    """(unclipped deltas, clipped deltas) as float32 from the device's own preq/postq: the target is formed in
    double from the clipped reward and max(postq) and stored as fp32, delta = preq[a] - target in fp32, and the
    clip (when clip > 0) follows the cost.  The reward is clipped as np.clip does, in double: the maximum with
    min_reward first, then the minimum with max_reward (crossed bounds give max_reward)."""
    preq, postq = np.asarray(preq, np.float32), np.asarray(postq, np.float32)
    raw = np.zeros_like(preq)
    for i, a in enumerate(actions):
        r = min(max(float(rewards[i]), float(min_reward)), float(max_reward))
        y = r if terminals[i] else r + float(discount) * float(postq[i].max())
        raw[i, a] = np.float32(preq[i, a]) - np.float32(y)
    clipped = np.clip(raw, np.float32(-clip), np.float32(clip)) if clip > 0 else raw.copy()
    return raw, clipped
