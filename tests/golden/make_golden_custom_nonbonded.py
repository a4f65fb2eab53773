"""Writes tests/golden/reference_custom_nonbonded.npz: the CustomNonbondedForce group of DHFR-LJ-table and DHFR-NBFIX
(tests/custom_nonbonded_harness.py) from the reference's own Reference platform (oracle/_ref): its energy (long-range
correction included), its forces, and the long-range coefficient CustomNonbondedForceImpl::calcLongRangeCorrection gives.
The positions are those of data/dhfr.npz rounded to fp32, which the harness rebuilds.

Run: python tests/golden/make_golden_custom_nonbonded.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import custom_nonbonded_harness as H  # noqa: E402


def main():
    out = {}
    for name, nbfix in (("lj_table", False), ("nbfix", True)):
        d, f = H.dhfr_lj_table(nbfix)
        s = H.Simulation(d, "Reference", forces=[f], pme=d.pme_parameters())
        forces, e = s.forces_energy(1 << H.CNB_GROUP)
        out[name + "_forces"] = forces
        out[name + "_energy"] = np.array(e)
        out[name + "_lrc"] = np.array(s.lrc())
        print("%-9s E = %.6f kJ/mol, long-range coefficient %.6f" % (name, e, out[name + "_lrc"]))
    np.savez_compressed(os.path.join(HERE, "reference_custom_nonbonded.npz"), **out)


if __name__ == "__main__":
    main()
