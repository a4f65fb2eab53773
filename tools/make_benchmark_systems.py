"""Builds the REAL benchmark systems of BASELINE.json (DHFR, ApoA1) as SystemDesc fixtures under data/, by running the
reference's own, unmodified Python application layer (wrappers/python/openmm/app: PDBFile, ForceField.createSystem,
forcefield.py 5k LoC) IN THIS CONTAINER against a thin recording stand-in for the SWIG module `openmm.openmm`
(the compiled wrapper cannot be built here: no swig/doxygen, SURVEY.md 8c).  Exactly the protocol of
examples/benchmark.py:97-138:

  dhfr  : amber99sb.xml + tip3p.xml on examples/5dfr_solv-cube_equil.pdb, PME, cutoff 0.9 nm, constraints=HBonds, rigid water
  apoa1 : amber14/protein.ff14SB + lipid17 + tip3p on examples/apoa1.pdb, PME, cutoff 1.0 nm, HBonds, hydrogenMass 1.5 amu
  dhfr_gbsa : amber99sb.xml + amber99_obc.xml on examples/5dfr_minimized.pdb, CutoffNonPeriodic, cutoff 2 nm, HBonds (the
              implicit-solvent protocol of examples/benchmark.py; the GBSA generator sets the reaction-field dielectric to 1)

The stand-in only RECORDS what forcefield.py builds (particles, bonds, angles, torsions, constraints, nonbonded
parameters); the one piece of C++ logic the application layer calls back into, NonbondedForce::createExceptionsFromBonds,
is executed by the real reference library (oracle/_ref, oracle.omm.exceptions_from_bonds).  Output: data/<name>.npz
(generated files are committed; /root/reference does not exist on the GPU box).

Run: python tools/make_benchmark_systems.py [dhfr] [apoa1] [dhfr_gbsa]   (dhfr_gbsa -> tests/golden/dhfr_gbsa.npz)
"""
import os
import sys
import types
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF_PY = "/root/reference/wrappers/python/openmm"
EXAMPLES = "/root/reference/examples"


def _install_mock():
    mm = types.ModuleType("openmm")
    mm.__path__ = [REF_PY]          # submodules (app, unit, vec3) come from the reference tree; its __init__ is not run
    sys.modules["openmm"] = mm
    import openmm.unit as unit      # noqa: E402  (pure python, from the reference)
    from openmm.vec3 import Vec3    # noqa: E402

    def s(x):
        if hasattr(x, "value_in_unit_system"):
            return x.value_in_unit_system(unit.md_unit_system)
        return x

    class Force(object):
        def __init__(self):
            self._group = 0
            self._periodic = False

        def setForceGroup(self, g):
            self._group = g

        def getForceGroup(self):
            return self._group

        def setUsesPeriodicBoundaryConditions(self, p):
            self._periodic = p

        def usesPeriodicBoundaryConditions(self):
            return self._periodic

    class System(object):
        def __init__(self):
            self.masses, self.constraints, self.forces, self.box = [], [], [], None

        def addParticle(self, m):
            self.masses.append(float(s(m)))
            return len(self.masses)-1

        def getNumParticles(self):
            return len(self.masses)

        def getParticleMass(self, i):
            return self.masses[i]*unit.dalton

        def setParticleMass(self, i, m):
            self.masses[i] = float(s(m))

        def addConstraint(self, i, j, d):
            self.constraints.append((int(i), int(j), float(s(d))))
            return len(self.constraints)-1

        def getNumConstraints(self):
            return len(self.constraints)

        def getConstraintParameters(self, k):
            i, j, d = self.constraints[k]
            return i, j, d*unit.nanometer

        def setDefaultPeriodicBoxVectors(self, a, b, c):
            self.box = np.array([[float(v) for v in s(a)], [float(v) for v in s(b)], [float(v) for v in s(c)]])

        def addForce(self, f):
            self.forces.append(f)
            return len(self.forces)-1

        def getNumForces(self):
            return len(self.forces)

        def getForce(self, i):
            return self.forces[i]

        def getForces(self):
            return list(self.forces)

        def isVirtualSite(self, i):
            return False

        def usesPeriodicBoundaryConditions(self):
            return True

    class HarmonicBondForce(Force):
        def __init__(self):
            Force.__init__(self)
            self.bonds = []

        def addBond(self, i, j, r0, k):
            self.bonds.append((int(i), int(j), float(s(r0)), float(s(k))))
            return len(self.bonds)-1

        def getNumBonds(self):
            return len(self.bonds)

        def getBondParameters(self, n):
            return self.bonds[n]

    class HarmonicAngleForce(Force):
        def __init__(self):
            Force.__init__(self)
            self.angles = []

        def addAngle(self, i, j, k, t0, kk):
            self.angles.append((int(i), int(j), int(k), float(s(t0)), float(s(kk))))
            return len(self.angles)-1

        def getNumAngles(self):
            return len(self.angles)

        def getAngleParameters(self, n):
            return self.angles[n]

    class PeriodicTorsionForce(Force):
        def __init__(self):
            Force.__init__(self)
            self.torsions = []

        def addTorsion(self, i, j, k, l, n, phase, kk):
            self.torsions.append((int(i), int(j), int(k), int(l), int(n), float(s(phase)), float(s(kk))))
            return len(self.torsions)-1

        def getNumTorsions(self):
            return len(self.torsions)

        def getTorsionParameters(self, n):
            return self.torsions[n]

    class NonbondedForce(Force):
        NoCutoff, CutoffNonPeriodic, CutoffPeriodic, Ewald, PME, LJPME = range(6)

        def __init__(self):
            Force.__init__(self)
            self.particles, self.exceptions = [], []
            self.method, self.cutoff, self.tol = 0, 1.0, 5e-4
            self.dispersion, self.switch, self.switch_distance = True, False, -1.0
            self.rf = 78.3

        def addParticle(self, q, sig, eps):
            self.particles.append([float(s(q)), float(s(sig)), float(s(eps))])
            return len(self.particles)-1

        def getNumParticles(self):
            return len(self.particles)

        def getParticleParameters(self, i):
            q, sg, ep = self.particles[i]
            return q*unit.elementary_charge, sg*unit.nanometer, ep*unit.kilojoule_per_mole

        def setParticleParameters(self, i, q, sig, eps):
            self.particles[i] = [float(s(q)), float(s(sig)), float(s(eps))]

        def addException(self, i, j, qq, sig, eps, replace=False):
            self.exceptions.append([int(i), int(j), float(s(qq)), float(s(sig)), float(s(eps))])
            return len(self.exceptions)-1

        def getNumExceptions(self):
            return len(self.exceptions)

        def getExceptionParameters(self, k):
            i, j, qq, sg, ep = self.exceptions[k]
            return i, j, qq*unit.elementary_charge**2, sg*unit.nanometer, ep*unit.kilojoule_per_mole

        def setExceptionParameters(self, k, i, j, qq, sig, eps):
            self.exceptions[k] = [int(i), int(j), float(s(qq)), float(s(sig)), float(s(eps))]

        def createExceptionsFromBonds(self, bonds, coulomb14, lj14):
            from oracle import omm
            p = np.array(self.particles)
            bi = np.array([b[0] for b in bonds], dtype=np.int32)
            bj = np.array([b[1] for b in bonds], dtype=np.int32)
            i, j, qq, sg, ep = omm.exceptions_from_bonds(p[:, 0], p[:, 1], p[:, 2], bi, bj, float(coulomb14), float(lj14))
            for k in range(len(i)):
                self.exceptions.append([int(i[k]), int(j[k]), float(qq[k]), float(sg[k]), float(ep[k])])

        def setNonbondedMethod(self, m):
            self.method = int(m)

        def getNonbondedMethod(self):
            return self.method

        def setCutoffDistance(self, c):
            self.cutoff = float(s(c))

        def setEwaldErrorTolerance(self, t):
            self.tol = float(t)

        def setUseDispersionCorrection(self, u):
            self.dispersion = bool(u)

        def setUseSwitchingFunction(self, u):
            self.switch = bool(u)

        def setSwitchingDistance(self, d):
            self.switch_distance = float(s(d))

        def setReactionFieldDielectric(self, d):
            self.rf = float(d)

        def setExceptionsUsePeriodicBoundaryConditions(self, p):
            pass

    class GBSAOBCForce(Force):
        NoCutoff, CutoffNonPeriodic, CutoffPeriodic = range(3)

        def __init__(self):
            Force.__init__(self)
            self.particles = []
            self.method, self.cutoff = 0, 1.0
            self.solute, self.solvent, self.surface = 1.0, 78.5, 2.25936

        def addParticle(self, q, radius, scale):
            self.particles.append([float(s(q)), float(s(radius)), float(s(scale))])
            return len(self.particles)-1

        def getNumParticles(self):
            return len(self.particles)

        def setNonbondedMethod(self, m):
            self.method = int(m)

        def setCutoffDistance(self, c):
            self.cutoff = float(s(c))

        def setSoluteDielectric(self, d):
            self.solute = float(d)

        def setSolventDielectric(self, d):
            self.solvent = float(d)

        def setSurfaceAreaEnergy(self, e):
            self.surface = float(s(e))

    class CMMotionRemover(Force):
        def __init__(self, frequency=1):
            Force.__init__(self)
            self.frequency = frequency

    class _Dummy(object):
        def __init__(self, *a, **k):
            pass

    for cls in (Force, System, HarmonicBondForce, HarmonicAngleForce, PeriodicTorsionForce, NonbondedForce, GBSAOBCForce, CMMotionRemover):
        setattr(mm, cls.__name__, cls)
    mm.Vec3 = Vec3

    def _getattr(name):           # every other SWIG class the app layer mentions at import time
        if name.startswith("__"):
            raise AttributeError(name)
        cls = type(name, (_Dummy,), {})
        setattr(mm, name, cls)
        return cls
    mm.__getattr__ = _getattr
    sub = types.ModuleType("openmm.openmm")
    sub.__getattr__ = lambda name: getattr(mm, name)
    sys.modules["openmm.openmm"] = sub
    mm.openmm = sub
    return mm, unit


def to_desc(system, positions_nm, name):
    from openmm_b200 import systems
    nb = [f for f in system.forces if type(f).__name__ == "NonbondedForce"]
    assert len(nb) == 1
    nb = nb[0]
    p = np.array(nb.particles)
    ex = np.array(nb.exceptions) if nb.exceptions else np.zeros((0, 5))
    d = systems.SystemDesc(masses=np.array(system.masses), charges=p[:, 0], sigmas=p[:, 1], epsilons=p[:, 2],
                           positions=np.asarray(positions_nm, dtype=np.float64), box=system.box, method=nb.method, cutoff=nb.cutoff,
                           ewald_tol=nb.tol, use_switch=nb.switch, switch_distance=max(nb.switch_distance, 0.0),
                           use_dispersion=nb.dispersion, rf_dielectric=nb.rf, name=name)
    d.exc_i, d.exc_j = ex[:, 0].astype(np.int32), ex[:, 1].astype(np.int32)
    d.exc_qq, d.exc_sigma, d.exc_eps = ex[:, 2].copy(), ex[:, 3].copy(), ex[:, 4].copy()
    bonds = [b for f in system.forces if type(f).__name__ == "HarmonicBondForce" for b in f.bonds]
    angles = [a for f in system.forces if type(f).__name__ == "HarmonicAngleForce" for a in f.angles]
    tors = [t for f in system.forces if type(f).__name__ == "PeriodicTorsionForce" for t in f.torsions]
    if bonds:
        b = np.array(bonds)
        d.bond_i, d.bond_j, d.bond_r0, d.bond_k = b[:, 0].astype(np.int32), b[:, 1].astype(np.int32), b[:, 2].copy(), b[:, 3].copy()
    if angles:
        a = np.array(angles)
        d.angle_i, d.angle_j, d.angle_k = a[:, 0].astype(np.int32), a[:, 1].astype(np.int32), a[:, 2].astype(np.int32)
        d.angle_t0, d.angle_kk = a[:, 3].copy(), a[:, 4].copy()
    if tors:
        t = np.array(tors)
        d.tor_i, d.tor_j, d.tor_k, d.tor_l = (t[:, k].astype(np.int32) for k in range(4))
        d.tor_n, d.tor_phase, d.tor_kk = t[:, 4].astype(np.int32), t[:, 5].copy(), t[:, 6].copy()
    if system.constraints:
        c = np.array(system.constraints)
        d.con_i, d.con_j, d.con_d = c[:, 0].astype(np.int32), c[:, 1].astype(np.int32), c[:, 2].copy()
    cm = [f for f in system.forces if type(f).__name__ == "CMMotionRemover"]
    d.cm_frequency = int(cm[0].frequency) if cm else 0
    gb = [f for f in system.forces if type(f).__name__ == "GBSAOBCForce"]
    if gb:
        g = np.array(gb[0].particles)
        d.gb_charges, d.gb_radii, d.gb_scales = g[:, 0].copy(), g[:, 1].copy(), g[:, 2].copy()
        d.gb_method = gb[0].method
        assert gb[0].method == NB_METHOD_OF_GB[nb.method] and (gb[0].method == 0 or gb[0].cutoff == nb.cutoff)
        d.gb_solute_dielectric, d.gb_solvent_dielectric, d.gb_surface_area_energy = gb[0].solute, gb[0].solvent, gb[0].surface
    return d


# GBSAOBCForce method that ForceField builds for each NonbondedForce method (forcefield.py GBSAOBCGenerator)
NB_METHOD_OF_GB = {0: 0, 1: 1, 2: 2, 3: 2, 4: 2}


def build(name):
    mm, unit = _install_mock()
    # openmm/app/internal/compiled.pyx (residue template matching) is Cython: compile it from where it lies into a
    # scratch build directory (the reference tree is read-only and is never written)
    import pyximport
    import tempfile
    pyximport.install(build_dir=os.path.join(tempfile.gettempdir(), "pyx_openmm_ref"), inplace=False, language_level=3)
    import openmm.app as app
    if name == "dhfr":
        pdb = app.PDBFile(os.path.join(EXAMPLES, "5dfr_solv-cube_equil.pdb"))
        ff = app.ForceField("amber99sb.xml", "tip3p.xml")
        system = ff.createSystem(pdb.topology, nonbondedMethod=app.PME, nonbondedCutoff=0.9*unit.nanometer, constraints=app.HBonds, rigidWater=True)
    elif name == "apoa1":
        pdb = app.PDBFile(os.path.join(EXAMPLES, "apoa1.pdb"))
        ff = app.ForceField("amber14/protein.ff14SB.xml", "amber14/lipid17.xml", "amber14/tip3p.xml")
        system = ff.createSystem(pdb.topology, nonbondedMethod=app.PME, nonbondedCutoff=1.0*unit.nanometer, constraints=app.HBonds, rigidWater=True,
                                 hydrogenMass=1.5*unit.amu)
    elif name == "dhfr_gbsa":
        pdb = app.PDBFile(os.path.join(EXAMPLES, "5dfr_minimized.pdb"))
        ff = app.ForceField("amber99sb.xml", "amber99_obc.xml")
        system = ff.createSystem(pdb.topology, nonbondedMethod=app.CutoffNonPeriodic, nonbondedCutoff=2.0*unit.nanometer, constraints=app.HBonds)
    else:
        raise SystemExit("unknown system " + name)
    pos = np.array(pdb.positions.value_in_unit(unit.nanometer))
    if system.box is None and pdb.topology.getPeriodicBoxVectors() is not None:
        v = pdb.topology.getPeriodicBoxVectors().value_in_unit(unit.nanometer)
        system.box = np.array([[float(x) for x in row] for row in v])
    d = to_desc(system, pos, name)
    out = os.path.join(ROOT, "tests", "golden") if name == "dhfr_gbsa" else os.path.join(ROOT, "data")
    os.makedirs(out, exist_ok=True)
    path = os.path.join(out, name + ".npz")
    d.save(path)
    print("%s: %d atoms, box %s, %d bonds %d angles %d torsions %d exceptions %d constraints, cm_freq %d -> %s (%.1f MB)" % (
        name, d.natoms, None if d.box is None else np.diag(d.box), len(d.bond_i), len(d.angle_i), len(d.tor_i), len(d.exc_i), len(d.con_i), d.cm_frequency, path,
        os.path.getsize(path)/1e6))
    return d


if __name__ == "__main__":
    for n in (sys.argv[1:] or ["dhfr"]):
        build(n)
