"""CPU half of the checkpoint tests: both rebuilt checkpoint layouts parse, and the numpy oracle reproduces the
stored Q-value KAT of the stand-in snapshot from them.  The device half is tests/test_gpu_checkpoint.py."""
import numpy as np
import pytest

from ckpt_helpers import fixture, write_checkpoint
from oracle import dqn_oracle as O


@pytest.mark.parametrize("layout", ["pre-1.0", "neon-1.3.0"])
def test_rebuilt_checkpoints_parse_and_reproduce_the_kat(tmp_path, layout):
    ws, ss, q_kat = fixture()
    path = str(tmp_path / "c.pkl")
    d = write_checkpoint(path, layout, ws, ss)
    if layout == "neon-1.3.0":
        assert d["neon_version"] == "1.3.0+344372b" and len(d["model"]["config"]["layers"]) == 9
    w2, s2 = O.load_snapshot(path)
    assert all((a == b).all() for a, b in zip(w2, ws)) and all((a == b).all() for a, b in zip(s2, ss))
    states = np.random.RandomState(1234).randint(0, 256, (32, 4, 84, 84)).astype(np.uint8)
    q = O.forward(w2, states)
    assert np.allclose(q[0], q_kat[0], atol=2e-5 * np.abs(q_kat).max())
    assert (q == q_kat).all()
