"""The persistent rollout kernel takes the cost's collision term from the graph build's neighbour scan: agent j collides
with i when acc < two_r_sq_thr, acc being the scan's squared distance, where the step cost asks 2r > sqrtf(acc).  The
kernel computes two_r_sq_thr once per rollout with sqrt_threshold(two_r) (geometry_dev.cuh), the device twin of
_lib.sqrt_threshold, and uses the flag only when 2r < comm_radius, which puts every agent closer than 2r in the row."""
import numpy as np
import pytest

F = np.float32


@pytest.mark.parametrize("env_id", ["SingleIntegrator", "DoubleIntegrator", "DubinsCar"])
def test_two_r_sq_thr_is_exact(env_id):
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.env import make_env
    d = make_env(env_id, 2, area_size=4.0, num_obs=0, device="cpu").desc(1, 0, edge_cap=64)
    two_r, rc = F(d.two_r), F(d.comm_radius)
    thr = F(_lib.sqrt_threshold(float(two_r)))
    # brute force over the 2 x 4096 fp32 values around (2r)^2 and thr
    for centre in (two_r * two_r, thr):
        b = np.array(centre, F).view(np.int32)
        x = (b + np.arange(-4096, 4097, dtype=np.int32)).view(F)
        assert np.array_equal(two_r > np.sqrt(x), x < thr), env_id
    assert np.sqrt(thr) >= two_r > np.sqrt(np.nextafter(thr, F(0)))
    # the flag is used in every 2-D environment, and every pair it flags is in the neighbour words
    assert two_r < rc and thr <= F(d.comm_sq_thr)
