"""Generates tests/golden/tile_forces.npz: the forces (and energies) of tests/test_gpu_sorted_forces.py's cases from the
tile kernel that still added its forces straight into the user-order force buffer, the version before the sorted-order
buffer and k_fold_sorted.  Needs a GPU.
Recipe: build libb200md.so of that version, then, from this tree,
    B200MD_LIB=<that build>/openmm_b200/libb200md.so python tests/golden/make_golden_tile_forces.py
Stored: f_<case> [atoms, 3] float64, exactly as Engine.get_forces returns it, and e_<case> (the potential energy, NaN
where the case evaluates forces only).
"""
import os
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main(out=os.path.join(HERE, "tile_forces.npz")):
    import test_gpu_sorted_forces as t
    res = {}
    for name in sorted(t.CASES):
        eng, f, e = t.run(name)
        res["f_" + name] = f
        res["e_" + name] = np.float64(np.nan if e is None else e)
        eng.close()
    np.savez_compressed(out, **res)
    print("%s (%s): %s" % (out, os.environ.get("B200MD_LIB", "this tree's build"), ", ".join("%s %d atoms" % (k[2:], len(v)) for k, v in res.items() if k[0] == "f")))


if __name__ == "__main__":
    main(*sys.argv[1:])
