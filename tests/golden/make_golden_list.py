"""Generates tests/golden/list_hashes.json: per case of tests/test_gpu_list_identity.py, the SHA-256 of the canonical
neighbour list, its tile and masked-tile counts, and the list builds so far, from the list kernels as they were before
they were reorganised (k_list_prep with a single-CTA scan, k_build_tiles searching every exclusion partner by bisection in
every tile).  Needs a GPU.
Recipe: build libb200md.so from this tree with that version's k_list_prep and k_build_tiles and their device helpers in
openmm_b200/csrc/nonbonded.cu (the read-back entry b200md_get_list is this tree's), then, from this tree,
    B200MD_LIB=<that build>/openmm_b200/libb200md.so python tests/golden/make_golden_list.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))


def main(out=os.path.join(HERE, "list_hashes.json")):
    import test_gpu_list_identity as t
    res = {}
    for name in t.CASES:
        eng, (digest, tiles, masked) = t.build(name)
        res[name] = {"sha256": digest, "tiles": tiles, "masked_tiles": masked, "list_builds": eng.stats()["list_builds"]}
        eng.close()
        print(name, res[name], flush=True)
    with open(out, "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
        f.write("\n")
    print("%s (%s)" % (out, os.environ.get("B200MD_LIB", "this tree's build")))


if __name__ == "__main__":
    main(*sys.argv[1:])
