"""Writes tests/golden/reference_gbsa.npz: energies and forces of a GBSAOBCForce alone, from the reference's own Reference
platform (oracle/_ref), for the cases the generalized Born tests pin the double-precision restatement (tests/gbsa_harness.py)
against:
  dhfr_nocutoff    the DHFR implicit-solvent fixture with both forces at NoCutoff
  dhfr_cutoff      the fixture as built: CutoffNonPeriodic, 2 nm
  hello_nacl       the six ions of the reference's HelloSodiumChloride example
  ion_box          400 ions in a 3.2 nm periodic box, CutoffPeriodic, 1.2 nm
  ion_box_custom   the same ions at NoCutoff, surface-area energy 0, dielectrics 4 and 40
  ion_box_tri_pmp  400 ions in the triclinic cell at the (+, -, +) limits of the reduced form, CutoffPeriodic 1.09 nm
  ion_box_tri_mpm  the same at the (-, +, -) limits
Each case stores the positions it was evaluated at and the GBSAOBCForce's energy and forces.

Run: python tests/golden/make_golden_gbsa.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import gbsa_harness as H  # noqa: E402


def main():
    out = {}
    for name, d in H.golden_cases().items():
        s = H.Simulation(d, "Reference")
        f, e = H.gb_only(s)
        out[name + "_positions"] = np.asarray(d.positions, dtype=np.float64)
        out[name + "_forces"] = f
        out[name + "_energy"] = np.array(e)
        print("%-15s %5d atoms  E = %.6f kJ/mol" % (name, d.natoms, e))
    np.savez_compressed(os.path.join(HERE, "reference_gbsa.npz"), **out)


if __name__ == "__main__":
    main()
