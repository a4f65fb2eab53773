"""Generates the committed golden fixtures of tests/golden/ from the reference sources and the oracle/_ref/ build of
them (so that the tests need neither).  Run: python tests/golden/make_golden.py

1. ewald_triclinic_gromacs.json -- the known-answer vector the reference's own test holds: 8 ions in a triclinic box,
   PME grid 32x40x48, alpha 3.45891, Gromacs forces and energy (tests/TestEwald.h:222-271; tolerance there 1e-4).
   Parsed from the header text, not retyped.
2. nacl_amorph.npz -- the 894-ion amorphous NaCl positions of tests/nacl_amorph.dat (used by tests/TestEwald.h:98-220)
   plus forces/energy of the reference's Reference platform (oracle/_ref/libOpenMM.so) with PME, cutoff 1.2,
   tol 1e-5 pinned to an FFT-friendly grid, and the Gromacs energy -3.82047e5 quoted by the test (Ewald, :150).
3. water5_reference.npz -- 375-atom TIP3P box: Reference-platform forces/energy (PME) for the seeded S1 recipe.
4. reference_platform.npz -- what the Reference platform computes for the inputs of tests/test_gpu_parity.py: forces
   (float32) and energy of every case of reference_cases() (above 512 atoms a sample: see _force_sample), the state
   after 10 deterministic steps of each integrator, and the DHFR constraints=AllBonds (CCMA) run on every atom of the
   CCMA network plus a seeded sample of the solvent;
   and, as "port_*" / "ccma_cpu:*", the Reference-platform results tests/test_oracle.py and tests/test_ccma_cpu.py hold
   the plain-C oracle to (float64).
"""
import json
import os
import re
import sys
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
REF = "/root/reference"


def parse_triclinic():
    src = open(os.path.join(REF, "tests/TestEwald.h")).read()
    blk = src[src.index("void testTriclinic()"):src.index("void testTriclinic2()")]
    vec = r"Vec3\(([^,]+),([^,]+),([^)]+)\)"
    box = [[float(x) for x in m] for m in re.findall(vec, re.search(r"setDefaultPeriodicBoxVectors\((.*)\);", blk).group(1))]
    pos = [[float(x) for x in m.groups()[1:]] for m in re.finditer(r"positions\[(\d)\] = " + vec, blk)]
    frc = [[float(x) for x in m.groups()[1:]] for m in re.finditer(r"expectedForce\[(\d)\] = " + vec, blk)]
    alpha, nx, ny, nz = re.search(r"setPMEParameters\(([^,]+),([^,]+),([^,]+),([^)]+)\)", blk).groups()
    energy = float(re.search(r"expectedEnergy = ([-0-9.e+]+)", blk).group(1))
    parts = re.findall(r"addParticle\(([-0-9.]+), ([0-9.]+), ([0-9.]+)\)", blk)
    assert len(pos) == 8 and len(frc) == 8 and len(parts) == 2
    out = {"source": "tests/TestEwald.h:222-271 (Gromacs)", "box": box, "positions": pos, "expected_forces": frc,
           "expected_energy": energy, "alpha": float(alpha), "grid": [int(nx), int(ny), int(nz)], "cutoff": 1.0,
           "charges": [float(parts[0][0])]*4 + [float(parts[1][0])]*4,
           "sigmas": [float(parts[0][1])]*4 + [float(parts[1][1])]*4,
           "epsilons": [float(parts[0][2])]*4 + [float(parts[1][2])]*4, "tolerance": 1e-4}
    json.dump(out, open(os.path.join(HERE, "ewald_triclinic_gromacs.json"), "w"), indent=1)
    return out


def nacl():
    from openmm_b200 import systems
    from oracle import omm
    txt = open(os.path.join(REF, "tests/nacl_amorph.dat")).read()
    pos = np.array([[float(x) for x in m] for m in re.findall(r"Vec3\(([^,]+),([^,]+),([^)]+)\)", txt)])
    assert pos.shape == (894, 3)
    # identical inputs for the fp32 device path and the double oracle: positions rounded to fp32-representable values
    # (rounding 3 nm coordinates moves them by <= 1.2e-7 nm, which alone changes ion-ion forces by ~2e-4 relative)
    pos = pos.astype(np.float32).astype(np.float64)
    n = 894
    L = 3.00646
    q = np.concatenate([np.ones(n//2), -np.ones(n//2)])
    d = systems.SystemDesc(masses=np.concatenate([np.full(n//2, 22.99), np.full(n//2, 35.45)]), charges=q, sigmas=np.ones(n), epsilons=np.zeros(n),
                           positions=pos, box=np.diag([L, L, L]), method=systems.NB_PME, cutoff=1.2, ewald_tol=1e-5, name="nacl_amorph")
    pme = d.pme_parameters()
    sim = omm.Simulation(d, "Reference", pme=pme)
    f, e = sim.forces_energy()
    np.savez_compressed(os.path.join(HERE, "nacl_amorph.npz"), positions=pos, box=L, charges=q, cutoff=1.2, ewald_tol=1e-5,
                        pme=np.array(pme), reference_forces=f, reference_energy=e, gromacs_energy=-3.82047e5)
    print("nacl_amorph: Reference PME energy %.3f (Gromacs Ewald %.3f), grid %s" % (e, -3.82047e5, pme))


def water():
    from openmm_b200 import systems
    from oracle import omm
    d = systems.water_box(5, cutoff=0.75).rounded()
    pme = d.pme_parameters()
    sim = omm.Simulation(d, "Reference", pme=pme)
    f, e = sim.forces_energy()
    np.savez_compressed(os.path.join(HERE, "water5_reference.npz"), positions=d.positions, pme=np.array(pme), reference_forces=f, reference_energy=e)
    print("water5: Reference energy %.4f" % e)


def _sample(n, k, seed=0):
    return np.arange(n, dtype=np.int32) if n <= k else np.sort(np.random.default_rng(seed).choice(n, k, replace=False)).astype(np.int32)


def _force_sample(omm, d, f, pme):
    """Above 512 atoms (10,000: the benchmark-size systems), a seeded sample of 512 (3,072) atoms plus the 256 (1,024) atoms
    most at risk in the floor-1 relative measure: those whose net force is smallest against the sum of its direct- and
    reciprocal-space parts, which is where fp32 errors of the large parts show (PME only; other methods: the sample)."""
    n = d.natoms
    if n <= 512:
        return np.arange(n, dtype=np.int32)
    k, k_risk = (512, 256) if n < 10000 else (3072, 1024)
    idx = set(_sample(n, k).tolist())
    if pme is not None:
        sim = omm.Simulation(d, "Reference", pme=pme, recip_group=1)
        f_dir, f_rec = sim.forces_energy(1)[0], sim.forces_energy(2)[0]
        risk = (np.linalg.norm(f_dir, axis=1) + np.linalg.norm(f_rec, axis=1))/np.maximum(1.0, np.linalg.norm(f, axis=1))
        idx |= set(np.argsort(-risk)[:k_risk].tolist())
    return np.array(sorted(idx), dtype=np.int32)


def reference_platform():
    from openmm_b200 import systems
    from oracle import omm
    sys.path.insert(0, os.path.dirname(HERE))
    import test_gpu_parity as t
    import test_ccma_cpu as c
    out = {}
    for name, d in t.reference_cases(systems).items():
        pme = d.pme_parameters() if d.method == systems.NB_PME else None
        f, e = omm.Simulation(d, "Reference", pme=pme).forces_energy()
        idx = _force_sample(omm, d, f, pme)
        out.update({name + ":idx": idx, name + ":xsum": d.positions.sum(), name + ":f": f[idx].astype(np.float32), name + ":e": e})
        print("%s: %d atoms, energy %.4f" % (name, d.natoms, e))
    d = systems.water_box(6, cutoff=0.9).rounded()
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.3
    for kind in (0, 1, 2):
        sim = omm.Simulation(d, "Reference", integrator=(kind, 0.0, 1.0, 0.001), pme=d.pme_parameters())
        sim.set_velocities(v)
        sim.step(10)
        st = sim.state(positions=True, velocities=True, energy=True)
        out.update({"integrate%d:dx" % kind: (st["positions"] - d.positions).astype(np.float32),
                    "integrate%d:v" % kind: st["velocities"].astype(np.float32), "integrate%d:kinetic" % kind: st["kinetic"]})
    d = t._all_bonds(systems, systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded())
    v = np.random.default_rng(3).standard_normal((d.natoms, 3))*0.2
    # every atom of a CCMA constraint (the protein) and a seeded sample of the rest (SETTLE waters)
    _, order, _, _, _ = c._probe(d.masses, d.con_i, d.con_j, d.con_d, (d.angle_i, d.angle_j, d.angle_k, d.angle_t0))
    net = np.unique(np.concatenate([d.con_i[order], d.con_j[order]]))
    rest = np.setdiff1d(np.arange(d.natoms), net)
    idx = np.sort(np.concatenate([net, rest[_sample(len(rest), 256, 2)]])).astype(np.int32)
    out["ccma:idx"] = idx
    for kind in (0, 1, 2):
        sim = omm.Simulation(d, "Reference", integrator=(kind, 0.0, 1.0, 0.001), constraint_tol=1e-6, pme=d.pme_parameters())
        sim.apply_constraints(1e-6)
        x0 = sim.state(positions=True)["positions"]
        if kind == 0:
            out["ccma:dx0"] = (x0[idx] - d.positions[idx]).astype(np.float32)
        sim.set_velocities(v)
        sim.step(10)
        out["ccma%d:dx" % kind] = (sim.state(positions=True)["positions"][idx] - d.positions[idx]).astype(np.float32)
        print("ccma kind %d done" % kind)
    out.update(reference_platform_cpu())
    np.savez_compressed(os.path.join(HERE, "reference_platform.npz"), **out)


def reference_platform_cpu():
    from openmm_b200 import systems
    from oracle import omm
    sys.path.insert(0, os.path.dirname(HERE))
    import test_oracle as t
    import test_ccma_cpu as c
    out = {}
    for name, d in t._cases():
        pme = d.pme_parameters() if d.method == systems.NB_PME else None
        out["port_%s:f" % name], out["port_%s:e" % name] = omm.Simulation(d, "Reference", pme=pme).forces_energy()
    d = systems.water_box(3, cutoff=0.45).rounded()
    for kind, friction in ((0, 0.0), (1, 0.0), (1, 5.0), (2, 0.0), (2, 5.0)):
        sim = omm.Simulation(d, "Reference", integrator=(kind, 0.0, friction, 0.002), pme=d.pme_parameters(), constraint_tol=1e-10)
        sim.step(5)
        st = sim.state(positions=True, velocities=True)
        key = "port_integrate%d_%g:" % (kind, friction)
        out[key + "x"], out[key + "v"] = st["positions"], st["velocities"]
    d = systems.water_box(3, cutoff=0.45, rigid=False).rounded()
    glob = {"lambda_q": 0.25, "lambda_lj": 1.0}
    p_off = [("lambda_q", 0, 0.3, 0.0, 0.0), ("lambda_q", 1, -0.3, 0.0, 0.0), ("lambda_lj", 3, 0.0, 0.02, 0.25), ("lambda_lj", 6, 0.1, -0.01, 0.5),
             ("lambda_q", 6, 0.05, 0.0, 0.0)]
    e_off = [("lambda_lj", 0, 0.04, 0.2, 0.3), ("lambda_q", 4, -0.02, 0.15, 0.1)]
    sim = omm.Simulation(d, "Reference", pme=d.pme_parameters(), nb_globals=glob, particle_offsets=p_off, exception_offsets=e_off)
    for k, values in enumerate((glob, {"lambda_q": -0.5, "lambda_lj": 0.4})):
        for name, value in values.items():
            sim.set_parameter(name, value)
        out["port_offsets%d:f" % k], out["port_offsets%d:e" % k] = sim.forces_energy()
    d = t._wrapped_chains()
    for tag, periodic in (("periodic", True), ("nonperiodic", False)):
        f, e = omm.Simulation(d, "Reference", pme=d.pme_parameters(), bonded_periodic=periodic).forces_energy()
        out["port_bonded_%s:f" % tag], out["port_bonded_%s:e" % tag] = f, e
    # DHFR, constraints=AllBonds, Context::applyConstraints(1e-7): the displacement of every atom up to the last one of a
    # CCMA constraint
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz"))
    d = __import__("test_gpu_parity")._all_bonds(systems, d)
    _, order, _, _, _ = c._probe(d.masses, d.con_i, d.con_j, d.con_d, (d.angle_i, d.angle_j, d.angle_k, d.angle_t0))
    k = int(max(d.con_i[order].max(), d.con_j[order].max())) + 1
    sim = omm.Simulation(d, "Reference", integrator=(systems.INT_VERLET, 0, 0, 0.001), constraint_tol=1e-7, pme=d.pme_parameters())
    sim.apply_constraints(1e-7)
    out["ccma_cpu:dx"] = (sim.state(positions=True)["positions"][:k] - d.positions[:k]).astype(np.float32)
    return out


if __name__ == "__main__":
    t = parse_triclinic()
    print("triclinic golden: E=%g, grid %s" % (t["expected_energy"], t["grid"]))
    nacl()
    water()
    reference_platform()
