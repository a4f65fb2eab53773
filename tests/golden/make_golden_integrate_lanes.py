"""Generates tests/golden/integrate_lanes.npz: 200-step trajectories of tests/test_gpu_integrate_lanes.py's mixed-unit system
(Verlet, Langevin and LangevinMiddle, single and mixed precision) from the integrate kernel that took one thread per
integration unit, the version of k_integrate before units were spread over one lane per atom.  Needs a GPU.
Recipe: check out that version, build it (python -c 'import __graft_entry__ as g; g.build()'), then
    python tests/golden/make_golden_integrate_lanes.py
Stored: x_<kind>_<precision>, v_<kind>_<precision> [atoms, 3] float64, exactly as Engine.get_positions/get_velocities
return them.
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main(out=os.path.join(HERE, "integrate_lanes.npz")):
    import test_gpu_integrate_lanes as t
    res = {}
    for kind in t.KINDS:
        for precision in ("single", "mixed"):
            x, v = t.run(kind, precision)
            res["x_%s_%s" % (kind, precision)] = x
            res["v_%s_%s" % (kind, precision)] = v
    np.savez_compressed(out, **res)
    print("%s: %d atoms, %d trajectories" % (out, len(x), len(res)//2))


if __name__ == "__main__":
    main(*sys.argv[1:])
