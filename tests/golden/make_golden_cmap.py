"""Generates tests/golden/charmm36_cmap.npz from the reference sources and the oracle/_ref/ build of them (so that the tests
need neither).  Run: python tests/golden/make_golden_cmap.py

The 8 CMAP maps of CHARMM36 (wrappers/python/openmm/app/data/charmm36.xml, <CMAPTorsionForce>), read as the reference's
ForceField reads them (the whitespace-separated energies of each <Map>, kJ/mol, size = sqrt of their number), and their
bicubic coefficients from CMAPTorsionForceImpl::calcMapDerivatives (tests/cmap_rb_harness.py coefficients):
    size [8], energy [8*24*24], coeff [8*24*24, 16].
"""
import os
import sys
import xml.etree.ElementTree as ET
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
REF = "/root/reference"


def main():
    import cmap_rb_harness
    tree = ET.parse(os.path.join(REF, "wrappers/python/openmm/app/data/charmm36.xml"))
    maps = [np.array([float(x) for x in m.text.split()]) for m in tree.getroot().find("CMAPTorsionForce").findall("Map")]
    size = np.array([int(round(np.sqrt(len(m)))) for m in maps], dtype=np.int32)
    assert all(s*s == len(m) for s, m in zip(size, maps))
    coeff = np.concatenate([cmap_rb_harness.coefficients(s, m) for s, m in zip(size, maps)])
    np.savez_compressed(os.path.join(HERE, "charmm36_cmap.npz"), size=size, energy=np.concatenate(maps), coeff=coeff)
    print("charmm36_cmap.npz: %d maps of size %s, %d patches" % (len(size), sorted(set(size.tolist())), len(coeff)))


if __name__ == "__main__":
    main()
