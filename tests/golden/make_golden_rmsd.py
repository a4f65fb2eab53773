"""Writes tests/golden/reference_rmsd.npz: the energy and forces of one RMSDForce alone, from the reference's own Reference
platform (oracle/_ref), for the cases of tests/rmsd_harness.py golden_cases():
  random_3 .. random_2000   random reference sets with perturbed copies
  mirror                    a mirror image of 60 points (its RMSD is not 0)
  rotated_copy              a rotated and translated copy (RMSD 0)
  offset_plus50/minus50     a perturbed, rotated copy moved by +-50 nm, as continuous coordinates can be
  subset, subset_all_listed 25 of the 60 particles, and all 60 listed explicitly (the all-particles case lists none)
Each case stores the positions, reference positions and particle list it was evaluated with.

Run: python tests/golden/make_golden_rmsd.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import rmsd_harness as H  # noqa: E402


def main():
    out = {}
    for name, (x, ref, particles) in H.golden_cases().items():
        e, f = H.evaluate(x, ref, particles, "Reference")
        out[name + "_positions"] = x
        out[name + "_reference"] = ref
        out[name + "_particles"] = particles
        out[name + "_energy"] = np.array(e)
        out[name + "_forces"] = f
        print("%-18s %5d particles  RMSD = %.9f nm" % (name, len(x), e))
    np.savez_compressed(os.path.join(HERE, "reference_rmsd.npz"), **out)


if __name__ == "__main__":
    main()
