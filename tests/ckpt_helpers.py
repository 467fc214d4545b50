"""Checkpoint fixtures shared by the CPU and GPU tests: a seeded stand-in for a trained snapshot and a writer that
rebuilds a checkpoint FILE with the reference's own pickle structure around any weights."""
import json
import os
import pickle

import numpy as np

from conftest import GOLDEN


def snapshot_weights(num_actions, seed=77):
    """Weights and RMSProp state of a snapshot's shapes, seeded: W ~ N(0, 2 / fan_in) (so Q values are O(1-10) like a
    trained net's), S = saturated second moments in [0, 1e-2).  (With S much smaller than g^2 the RMSProp step is ~sign(g)
    and two correct fp32 implementations drift apart by percents within 5 steps.)"""
    from oracle import dqn_oracle as O
    rs = np.random.RandomState(seed)
    ws, ss = [], []
    for shp in O.layer_shapes(num_actions):
        ws.append((rs.standard_normal(shp) * np.sqrt(2.0 / shp[0])).astype(np.float32))
        ss.append((rs.random_sample(shp) * 1e-2).astype(np.float32))
    return ws, ss


def fixture():
    """(W, S) of the A = 4 stand-in snapshot and q_kat: the numpy oracle's Q rows for it on the KAT states
    (RandomState(1234) uint8 states), stored when the fixture was made (tests/golden/make_snapshot_fixture.py)."""
    ws, ss = snapshot_weights(4)
    return ws, ss, np.load(os.path.join(GOLDEN, "snapshot_q_kat.npz"))["q_kat"]


def rebuild(skel, arrays):
    """Inverse of make_snapshot_fixture.skeleton(): arrays are consumed in traversal order."""
    if isinstance(skel, dict):
        if skel.get("__ndarray__"):
            a = next(arrays)
            assert list(a.shape) == skel["shape"] or skel["shape"][0] == 18, (a.shape, skel["shape"])
            return a
        if "__seq__" in skel:
            items = [rebuild(v, arrays) for v in skel["items"]]
            return tuple(items) if skel["__seq__"] == "tuple" else items
        return {k: rebuild(v, arrays) for k, v in skel.items()}
    return skel


def write_checkpoint(path, layout, ws, ss):
    """A checkpoint file with the reference's own structure (keys, nesting, type strings) around (ws, ss)."""
    meta = json.load(open(os.path.join(GOLDEN, "snapshot_layouts.json")))
    skel = meta["breakout_77" if layout == "pre-1.0" else "seaquest_178"]["skeleton"]
    order = []
    if layout == "pre-1.0":
        for w, s in zip(ws, ss):            # dict traversal order of the skeleton: params before states
            order += [w, s]
        d = rebuild(skel, iter(order))
    else:
        # json sorted the keys: inside a layer dict "params" precedes "states"
        for w, s in zip(ws, ss):
            order += [w, s]
        d = rebuild(skel, iter(order))
        d["model"]["config"]["layers"][-1]["config"]["nout"] = int(ws[4].shape[0])
    with open(path, "wb") as f:
        pickle.dump(d, f, protocol=2)
    return d


