"""Generate the 256-sample golden fixtures FROM THE REFERENCE ITSELF (same recipe as make_golden.py).

Run with a checkout of the reference (MIPNERF_REFERENCE=<path>):

    python tests/golden/make_golden_samples256.py

A ray of 256 samples is two 128-row tiles in the tensor-core level kernel.  Two fixtures:
  * forward_n256.npz: num_samples=256, trained_like weights, 32 multiscale rays, deterministic, black background,
    with the fine level's searchsorted indices;
  * forward_n256_randomized.npz: 16 rays, randomized, density_noise=1.0, the generator's draws (t_rand, u_jitter and
    the density normals of both levels) replayed into the fixture.
Only the reference's numerical outputs are recorded (provenance: VERSIONS_samples256.txt).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from make_golden import forward_case  # noqa: E402  (imports the reference from MIPNERF_REFERENCE)


def samples256_case():
    forward_case("forward_n256.npz", 32, seed=7, weights_kind="trained_like", randomized=False, white_bkgd=False,
                 multiscale=True, num_samples=256)
    forward_case("forward_n256_randomized.npz", 16, seed=8, weights_kind="trained_like", randomized=True,
                 white_bkgd=True, num_samples=256, density_noise=1.0)


if __name__ == "__main__":
    samples256_case()
