"""oracle/ref_cpu_path.py (the torch-CPU restatement timed as the CPU baseline) against the real reference's recorded
trajectories (tests/golden)."""

import os
import numpy as np
import pytest
from oracle.ref_cpu_path import PGPEReferencePath

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("tag,sense", [("pgpe", "min"), ("pgpe_max", "max")])
def test_port_reproduces_golden_trajectory(golden, tag, sense):
    p = PGPEReferencePath(8, 32, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0, seed=11, sense=sense)
    for t in range(len(golden[f"traj/{tag}/mu"])):
        p.step()
        np.testing.assert_allclose(p.mu.numpy(), golden[f"traj/{tag}/mu"][t], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(p.sigma.numpy(), golden[f"traj/{tag}/sigma"][t], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(p.X.numpy(), golden[f"traj/{tag}/X"][t], rtol=1e-6, atol=2e-6)


def test_port_is_bit_identical_to_the_reference():
    """The reference's own PGPE run (tests/golden/gen_ref_cpu_port_golden.py), generation by generation, bit for bit."""
    with np.load(os.path.join(ROOT, "tests", "golden", "ref_cpu_port_golden.npz")) as z:
        ref = {k: z[k] for k in z.files}
    p = PGPEReferencePath(300, 200, center_learning_rate=0.5, stdev_learning_rate=0.1, stdev_init=1.0, seed=5)
    for t in range(len(ref["mu"])):
        p.step()
        assert np.array_equal(p.mu.numpy(), ref["mu"][t]), t
        assert np.array_equal(p.sigma.numpy(), ref["sigma"][t]), t
        if t == 0:
            assert np.array_equal(p.X.numpy(), ref["X_first"])
    assert np.array_equal(p.X.numpy(), ref["X_last"])
