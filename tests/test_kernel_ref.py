"""Calibration of tests/kernel_ref.py on the CPU: the f64 layers agree with the oracle, the emulated hi/lo scheme
stays at least 4× inside the bound at every batch of the GPU sweep, and each way of getting the scheme subtly wrong
exceeds it; for the scalar net and for the dueling net, whose fc1 is 1024 wide.  Run with -s to see the table: per batch and kernel, the scheme's margin (bound / worst error) and the
worst ratio of error to bound under each mutation ("-" where a kernel has no such part)."""
import numpy as np
import pytest

import dueling_oracle as D
import kernel_ref as K
from oracle import dqn_oracle as O

SWEEP = [1, 2, 3, 16, 33, 63, 64, 65, 128, 129, 256, 257, 512]
F32 = np.float32
MUTATIONS = ["A_lo dropped", "B_lo dropped", "lo x 2^10", "k-block skipped", "split dropped", "last row zeroed",
             "stale lo"]
# the dueling net's fc1 is two 512-unit streams side by side: fc1_fwd losing m-tiles 4-7 (the value stream's units),
# fc1_dgrad reducing over only 8 of its 16 k-blocks
DUELING_MUTATIONS = MUTATIONS + ["one stream dropped"]


def _operands(batch, seed=2, dueling=False):
    """The operands each kernel sees in one training step of a Q-of-order-1 network (fc weights × 3, as the GPU
    tests use), with dZ formed in f64 and stored as fp32 like the kernels store it; plus the weights after one
    RMSProp step from zero state (a stale-lo image is the old weights' lo plane).  dueling: the dueling net, fc1
    (1024, 3136) and fc2 (A + 1, 512), with dZ4 from the dueling head's rule 3 on its deltas."""
    ws = (D.xavier_init if dueling else O.xavier_init)(4, seed)
    ws[3] = ws[3] * F32(3)
    ws[4] = ws[4] * F32(3)
    rs = np.random.RandomState(seed)
    pre = rs.randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    post = rs.randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    act = rs.randint(0, 4, batch)
    rew = rs.randint(-3, 4, batch)
    term = rs.rand(batch) < 0.3
    fwd = D.forward if dueling else O.forward
    q, acts = fwd(ws, pre, keep=True)
    _, d = K.head_td(q, fwd(ws, post), act, rew, term)
    h1, h2, h3, h4 = acts["h1"], acts["h2"], acts["h3"], acts["h4"]
    if dueling:
        dz4 = D.dz4(h4, ws[4], *D.stream_grads(d[np.arange(batch), act], act, 4))
    else:
        dz4 = ((d @ ws[4]) * (h4 > 0)).astype(F32)
    dz3 = (K.fc_dgrad(dz4, ws[3]).reshape(batch, 64, 7, 7) * (h3 > 0)).astype(F32)
    dz2 = (K.conv_dgrad(2)(dz3, ws[2]) * (h2 > 0)).astype(F32)
    dz1 = (K.conv_dgrad(1)(dz2, ws[1]) * (h1 > 0)).astype(F32)
    grads = [K.conv_wgrad(0)(K.states_f64(pre), dz1), K.conv_wgrad(1)(h1, dz2), K.conv_wgrad(2)(h2, dz3),
             K.fc_wgrad(h3, dz4)]
    new = [w.copy() for w in ws[:4]]
    O.rmsprop_update(new, [np.zeros_like(w) for w in new], [g.astype(F32) for g in grads], batch)
    x = (pre.astype(F32) / F32(255)).astype(F32)
    return dict(x=x, h1=h1, h2=h2, h3=h3, dz1=dz1, dz2=dz2, dz3=dz3, dz4=dz4, w=ws, new=new)


def _zero(t, index):
    t = np.array(t, copy=True)
    t[index] = 0
    return t


def _kernels(o, batch):
    """(name, op, A, B, A exact, weight-operand index or None, k-block skip, split drop, zero last M row).
    The skips zero one operand's slice of the reduction: the last k-block, or the last split's k-blocks."""
    w, n = o["w"], batch
    hidden = w[3].shape[0]

    def pix(t, lo, hi):                  # reduction over output pixels (n, p, q) in order: zero dZ rows [lo, hi)
        flat = np.ascontiguousarray(np.asarray(t).transpose(0, 2, 3, 1)).reshape(-1, t.shape[1])
        flat = _zero(flat, slice(lo, hi))
        return flat.reshape(t.shape[0], t.shape[2], t.shape[3], t.shape[1]).transpose(0, 3, 1, 2)

    def tap_rows(layer, kb):             # conv forward: k-block kb of the internal (r, s, c) order, as Neon rows
        r, s, _, _ = K.CONV[layer]
        c = w[layer].shape[0] // (r * s)
        ks = np.arange(kb * 64, kb * 64 + 64)
        rr, ss, cc = ks // (s * c), (ks // c) % s, ks % c
        return cc * r * s + rr * s + ss

    ks = []
    # forward: A = activations, B = weights
    ks.append(("conv1_fwd", K.conv_fwd(0), o["x"], w[0], True, 1,
               lambda: (o["x"], _zero(w[0], slice(192, 256))), None, lambda y: _zero(y, (-1, slice(None), -1, -1))))
    ks.append(("conv2_fwd", K.conv_fwd(1), o["h1"], w[1], False, 1,
               lambda: (o["h1"], _zero(w[1], tap_rows(1, 7))), None, lambda y: _zero(y, (-1, slice(None), -1, -1))))
    ks.append(("conv3_fwd", K.conv_fwd(2), o["h2"], w[2], False, 1,
               lambda: (o["h2"], _zero(w[2], tap_rows(2, 8))), None, lambda y: _zero(y, (-1, slice(None), -1, -1))))
    sp = K.fc1_splits(n)
    per = -(-49 // sp)
    fc1_cols = lambda kb0, kb1: (np.arange(64)[:, None] * 49 + np.arange(kb0, kb1)[None, :]).ravel()
    ks.append(("fc1_fwd", K.fc_fwd, o["h3"], w[3], False, 1,
               lambda: (o["h3"], _zero(w[3], (slice(None), fc1_cols(48, 49)))),
               lambda sp=sp, per=per: (o["h3"], _zero(w[3], (slice(None), fc1_cols((sp - 1) * per, 49)))),
               lambda y: _zero(y, (slice(None), -1))))
    # data gradients: A = dZ, B = weights
    fc1_dgrad = lambda a, b: K.fc_dgrad(a, b).reshape(len(a), 64, 7, 7)
    ks.append(("fc1_dgrad", fc1_dgrad, o["dz4"], w[3], False, 1,
               lambda: (o["dz4"], _zero(w[3], slice(hidden - 64, hidden))), None,
               lambda y: _zero(y, (slice(None), 63, 6, 6))))
    ks.append(("conv3_dgrad", K.conv_dgrad(2), o["dz3"], w[2], False, 1,
               lambda: (o["dz3"], _zero(w[2], np.arange(64) * 9 + 8)), None,
               lambda y: _zero(y, (-1, slice(None), -1, -1))))
    ks.append(("conv2_dgrad", K.conv_dgrad(1), o["dz2"], w[1], False, 1,
               lambda: (o["dz2"], _zero(w[1], np.arange(32) * 16 + 15)), None,
               lambda y: _zero(y, (-1, slice(None), -1, -1))))
    # weight gradients: A = activations, B = dZ; the reduction runs over pixels (or samples for fc1)
    nb = -(-n // 64)
    ks.append(("fc1_wgrad", K.fc_wgrad, o["h3"], o["dz4"], False, None,
               lambda: (o["h3"], _zero(o["dz4"], slice((nb - 1) * 64, n))), None,
               lambda y: _zero(y, (slice(None), -1))))
    for layer, name, a, b in ((2, "conv3_wgrad", o["h2"], o["dz3"]), (1, "conv2_wgrad", o["h1"], o["dz2"]),
                              (0, "conv1_wgrad", o["x"], o["dz1"])):
        pixels = n * (400, 81, 49)[layer]
        per, sp = K.wgrad_split(layer, n)
        kbs = -(-pixels // 64)
        ks.append((name, K.conv_wgrad(layer), a, b, layer == 0, None,
                   (lambda a=a, b=b, kbs=kbs, pixels=pixels: (a, pix(b, (kbs - 1) * 64, pixels))),
                   (lambda a=a, b=b, per=per, sp=sp, pixels=pixels: (a, pix(b, (sp - 1) * per * 64, pixels)))
                   if sp > 1 else None,
                   lambda y: _zero(y, -1)))
    return ks


def _calibrate(batch, dueling=False):
    o = _operands(batch, dueling=dueling)
    hidden = o["w"][3].shape[0]
    rows = {}
    for name, op, a, b, exact, widx, skip, drop, zero_row in _kernels(o, batch):
        y = op(np.asarray(a, np.float64), np.asarray(b, np.float64))
        bnd = K.bound(op, a, b, K.chain(name, batch, hidden=hidden), y, a_exact=exact)
        emu = lambda **kw: K.gemm_hilo(op, a, b, a_exact=exact, **kw)
        r = {"scheme": K.ratio(emu(), y, bnd)}
        if name in ("conv1_wgrad", "conv2_wgrad", "conv3_wgrad", "fc1_wgrad"):
            # fp32 accumulation in k-block and split-K order, on the GEMM the kernel runs
            layer = {"conv1_wgrad": 0, "conv2_wgrad": 1, "conv3_wgrad": 2}.get(name)
            if layer is None:
                cols, rws, per, sp = np.asarray(a).reshape(batch, -1), b, -(-batch // 64), 1
            else:
                cols = K.im2col(np.asarray(a, np.float64), layer)[0]
                rws = np.asarray(b).transpose(0, 2, 3, 1).reshape(-1, np.asarray(b).shape[1])
                per, sp = K.wgrad_split(layer, batch)
            g = K.wgrad_fp32_chunked(cols, rws, per, sp, a_exact=exact)
            r["scheme"] = max(r["scheme"], K.ratio(g.T if layer is None else g, y, bnd))
        r["A_lo dropped"] = None if exact else K.ratio(emu(drop_a_lo=True), y, bnd)
        r["B_lo dropped"] = K.ratio(emu(drop_b_lo=True), y, bnd)
        r["lo x 2^10"] = K.ratio(emu(lo_scale=2.0 ** 10), y, bnd)
        r["k-block skipped"] = K.ratio(K.gemm_hilo(op, *skip(), a_exact=exact), y, bnd)
        r["split dropped"] = None if drop is None else K.ratio(K.gemm_hilo(op, *drop(), a_exact=exact), y, bnd)
        r["last row zeroed"] = K.ratio(zero_row(emu()), y, bnd)
        if widx is None:
            r["stale lo"] = None
        else:   # the kernel multiplies the updated weights' hi plane by the old weights' lo plane
            layer = {"conv1_fwd": 0, "conv2_fwd": 1, "conv3_fwd": 2, "fc1_fwd": 3, "fc1_dgrad": 3,
                     "conv3_dgrad": 2, "conv2_dgrad": 1}[name]
            wn = o["new"][layer]
            yn = op(np.asarray(a, np.float64), np.asarray(wn, np.float64))
            bn = K.bound(op, a, wn, K.chain(name, batch, hidden=hidden), yn, a_exact=exact)
            r["stale lo"] = K.ratio(K.gemm_hilo(op, a, wn, a_exact=exact, b_lo_from=b), yn, bn)
        if not dueling:
            r["one stream dropped"] = None
        elif name == "fc1_fwd":       # m-tiles 4-7 (128 units each) never written: the value stream's units read 0
            r["one stream dropped"] = K.ratio(_zero(emu(), (slice(None), slice(hidden // 2, None))), y, bnd)
        elif name == "fc1_dgrad":     # k-blocks 8-15 (the value stream's units) left out of the reduction
            r["one stream dropped"] = K.ratio(K.gemm_hilo(op, a, _zero(b, slice(hidden // 2, None))), y, bnd)
        else:
            r["one stream dropped"] = None
        rows[name] = r
    return rows


def _report_and_assert(batch, rows, mutations, hidden):
    print("\nbatch %d  %s" % (batch, K.dispatch(batch, hidden=hidden)))
    print("  %-12s %8s  " % ("kernel", "margin") + "  ".join("%15s" % m for m in mutations))
    for name, r in rows.items():
        print("  %-12s %7.0fx  " % (name, 1 / max(r["scheme"], 1e-30)) +
              "  ".join("%15s" % ("-" if r[m] is None else "%.3g" % r[m]) for m in mutations))
    for name, r in rows.items():
        assert r["scheme"] <= 0.25, (name, r["scheme"])
        for m in mutations:
            assert r[m] is None or r[m] > 1.0, (name, m, r[m])


@pytest.mark.parametrize("batch", SWEEP)
def test_bound_separates_the_scheme_from_its_mutations(batch):
    _report_and_assert(batch, _calibrate(batch), MUTATIONS, K.HIDDEN)


@pytest.mark.parametrize("batch", SWEEP)
def test_bound_separates_the_dueling_scheme_from_its_mutations(batch):
    """The dueling net: fc1 1024 wide (fc1_dgrad's chain doubles), W5 (A + 1, 512), dZ4 from the dueling head's
    stream gradients.  Every kernel, the three fc1 kernels at width 1024 among them, stays 4× inside the bound, and
    each mutation, dropping one of the two streams included, exceeds it."""
    rows = _calibrate(batch, dueling=True)
    for name in ("fc1_fwd", "fc1_dgrad"):
        assert rows[name]["one stream dropped"] is not None
    _report_and_assert(batch, rows, DUELING_MUTATIONS, 2 * K.HIDDEN)


def test_dispatch_of_the_sweep():
    """The sweep reaches both conv2/conv3 forward paths, both fc1 split counts and the conv weight gradients from one
    split up to the 48 k_opt_conv reduces."""
    d = [K.dispatch(b) for b in SWEEP]
    assert {x["conv23"] for x in d} == {True, False}
    assert {x["fc1_splits"] for x in d} == {7, 4}
    assert min(min(x["wgrad_splits"]) for x in d) == 1 and max(max(x["wgrad_splits"]) for x in d) == 48
    assert K.dispatch(64)["conv23"] and not K.dispatch(65)["conv23"]
    assert K.dispatch(256)["fc1_splits"] == 7 and K.dispatch(257)["fc1_splits"] == 4


@pytest.mark.parametrize("batch", [1, 5])
def test_f64_layers_agree_with_the_oracle(batch):
    """The f64 layers restate the oracle's fp32 forward and backward (oracle/dqn_oracle.py)."""
    ws = O.xavier_init(4, 1)
    rs = np.random.RandomState(batch)
    pre = rs.randint(0, 256, (batch, 4, 84, 84)).astype(np.uint8)
    q, acts = O.forward(ws, pre, keep=True)
    h1 = K.relu(K.conv_fwd(0)(K.states_f64(pre), ws[0]))
    h2 = K.relu(K.conv_fwd(1)(h1, ws[1]))
    h3 = K.relu(K.conv_fwd(2)(h2, ws[2]))
    h4 = K.relu(K.fc_fwd(h3, ws[3]))
    for mine, ref in ((h1, acts["h1"]), (h2, acts["h2"]), (h3, acts["h3"]), (h4, acts["h4"]),
                      (K.fc_fwd(h4, ws[4]), q)):
        assert np.abs(mine - ref).max() <= 1e-5 * np.abs(ref).max()
    d = rs.randn(batch, 4).astype(F32)
    grads = O.backward(ws, acts, d)
    dz4 = K.fc_dgrad(d, ws[4]) * (acts["h4"] > 0)
    dz3 = K.fc_dgrad(dz4, ws[3]).reshape(batch, 64, 7, 7) * (acts["h3"] > 0)
    dz2 = K.conv_dgrad(2)(dz3, ws[2]) * (acts["h2"] > 0)
    dz1 = K.conv_dgrad(1)(dz2, ws[1]) * (acts["h1"] > 0)
    mine = [K.conv_wgrad(0)(K.states_f64(pre), dz1), K.conv_wgrad(1)(acts["h1"], dz2),
            K.conv_wgrad(2)(acts["h2"], dz3), K.fc_wgrad(acts["h3"], dz4), K.fc_wgrad(acts["h4"], d)]
    for l, (g, ref) in enumerate(zip(mine, grads)):
        assert np.abs(g - ref).max() <= 1e-4 * np.abs(ref).max(), l


def test_split_rounds_like_the_device():
    """hi/lo as __float2half_rn writes them: nearest even, subnormal lo kept, and hi + lo·2⁻¹¹ within 2⁻²²|x| + 2⁻³⁶."""
    rs = np.random.RandomState(0)
    x = np.concatenate([rs.randn(4096), rs.randn(4096) * 1e-6, rs.randn(4096) * 1e-9, [0.0, 1.0, 2 ** -24]]).astype(F32)
    hi, lo = K.split(x)
    rec = hi.astype(np.float64) + lo.astype(np.float64) / K.LO_SCALE
    assert (np.abs(rec - x) <= 2.0 ** -22 * np.abs(x) + 2.0 ** -36).all()
    assert (lo[np.abs(x) < 1e-7] != 0).any()                      # subnormal lo planes are kept, not flushed
    assert K.split(np.array([1 + 2 ** -11], F32))[0][0] == 1.0    # a tie rounds to even
