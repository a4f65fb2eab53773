"""Writes tests/golden/reference_barostat.npz for tests/test_gpu_barostat.py: the Reference platform's forces and energy of
DHFR and ApoA1 after a barostat move (ReferenceMonteCarloBarostat::applyBarostat, restated in tests/barostat_harness.py,
scale BAROSTAT_SCALE on every axis) in the scaled box, on the atom sample of make_golden._force_sample; and the scaled
positions of that sample.  Needs oracle/_ref/.  Run: python tests/golden/make_golden_barostat.py"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, HERE, os.path.dirname(HERE)]
BAROSTAT_SCALE = 1.02


def main():
    from openmm_b200 import systems
    from oracle import omm
    from make_golden import _force_sample
    from barostat_harness import barostat_scale
    out = {}
    for name in ("dhfr", "apoa1"):
        d = systems.SystemDesc.load(os.path.join(ROOT, "data", name + ".npz")).rounded()
        x = barostat_scale(d.positions, d.molecules(), d.box, (BAROSTAT_SCALE,)*3).astype(np.float32).astype(np.float64)
        pme = d.pme_parameters()
        ds = systems.SystemDesc(**{**d.__dict__, "positions": x, "box": d.box*BAROSTAT_SCALE})
        f, e = omm.Simulation(ds, "Reference", pme=pme).forces_energy()
        idx = _force_sample(omm, ds, f, pme)
        out.update({name + ":idx": idx, name + ":x": x[idx].astype(np.float32), name + ":f": f[idx].astype(np.float32), name + ":e": e})
        print("barostat %s: energy %.4f" % (name, e))
    np.savez_compressed(os.path.join(HERE, "reference_barostat.npz"), **out)


if __name__ == "__main__":
    main()
