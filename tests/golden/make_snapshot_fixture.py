"""Generate tests/golden/snapshot_q_kat.npz and, given the reference's shipped checkpoints (SNAP below),
snapshot_layouts.json:

    python tests/golden/make_snapshot_fixture.py [--layouts]

What is kept (data only — no reference source):
  * snapshot_q_kat.npz: the fp32 Q-values the numpy oracle computes on the KAT input of SURVEY §8(c)
    (RandomState(1234) states) from the seeded stand-in snapshot of tests/ckpt_helpers.py — the known answer
    the device must reproduce.  (A trained snapshot's weights are 13 MB, too large to keep as test data.)
  * --layouts: the SKELETONS of breakout_77.pkl (pre-1.0 ``layer_params_states`` layout) and seaquest_178.pkl
    (neon 1.3.0 layout) — every key, type string and config dict with the arrays replaced by (shape, dtype,
    crc32) — so that tests can rebuild a byte-faithful checkpoint in either layout around any weights and check
    that the product's writer emits the same structure.
"""
import json
import os
import pickle
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
SNAP = "/root/reference/snapshots"

from oracle import dqn_oracle as O  # noqa: E402


def crc(a):
    return int(zlib.crc32(np.ascontiguousarray(a).tobytes()) & 0xffffffff)


def skeleton(obj):
    """The structure of a checkpoint with every ndarray replaced by a descriptor."""
    if isinstance(obj, np.ndarray):
        return {"__ndarray__": True, "shape": list(obj.shape), "dtype": str(obj.dtype), "crc32": crc(obj)}
    if isinstance(obj, dict):
        return {str(k): skeleton(v) for k, v in obj.items()}
    if isinstance(obj, (list, tuple)):
        return {"__seq__": type(obj).__name__, "items": [skeleton(v) for v in obj]}
    if isinstance(obj, (np.integer,)):
        return int(obj)
    if isinstance(obj, (np.floating,)):
        return float(obj)
    if isinstance(obj, bytes):
        return obj.decode("latin1")
    return obj


def main():
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from ckpt_helpers import snapshot_weights
    ws, _ = snapshot_weights(4)
    states = np.random.RandomState(1234).randint(0, 256, (32, 4, 84, 84)).astype(np.uint8)
    np.savez_compressed(os.path.join(HERE, "snapshot_q_kat.npz"), q_kat=O.forward(ws, states).astype(np.float32))
    if "--layouts" not in sys.argv:
        return
    with open(os.path.join(SNAP, "breakout_77.pkl"), "rb") as f:
        old = pickle.load(f, encoding="latin1")
    with open(os.path.join(SNAP, "seaquest_178.pkl"), "rb") as f:
        new = pickle.load(f, encoding="latin1")
    new = dict(new)
    new["backend"] = {k: v for k, v in new["backend"].items() if k != "rng_state"}   # 0.8 MB of RNG words: dropped
    meta = {"breakout_77": {"layout": "pre-1.0 layer_params_states", "skeleton": skeleton(old)},
            "seaquest_178": {"layout": "neon 1.3.0", "skeleton": skeleton(new),
                             "note": "backend.rng_state (NervanaGPU RNG words) omitted from the skeleton"}}
    with open(os.path.join(HERE, "snapshot_layouts.json"), "w") as f:
        json.dump(meta, f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main()
