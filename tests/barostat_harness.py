"""Test infrastructure for the Monte Carlo barostat (tests/test_oracle_barostat.py, tests/test_gpu_barostat.py,
tests/golden/make_golden_barostat.py):

- barostat_scale: ReferenceMonteCarloBarostat::applyBarostat (ReferenceMonteCarloBarostat.cpp:67-103) restated in double;
- run_npt: a SystemDesc as the reference's System XML, run with a barostat on any platform by plugin/examples/run_npt.cpp
  (built into oracle/_ref/tests where the reference sources are present)."""
import json
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RUN_NPT = os.path.join(ROOT, "oracle", "_ref", "tests", "run_npt")
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")


def barostat_scale(positions, molecules, box, scale):
    """Every molecule's centre (unweighted mean, :79-84; Vec3::operator/= multiplies by the reciprocal) is moved into the first
    periodic box along c, then b, then a (:88-91), scaled per axis (:95-97), and every atom of the molecule moves by the
    difference (:98-102).  Returns the new positions [N,3]."""
    x = np.array(positions, dtype=np.float64)
    box = np.asarray(box, dtype=np.float64)
    s = np.asarray(scale, dtype=np.float64)
    for m in molecules:
        c = np.zeros(3)
        for a in m:
            c = c + x[a]
        c = c*(1.0/len(m))
        p = c.copy()
        for v in (2, 1, 0):
            p = p - box[v]*np.floor(p[v]/box[v][v])
        x[m] += p*s - c
    return x


def run_npt(desc, workdir, platform="B200", pme=None, timeout=1200, **options):
    """Run desc with plugin/examples/run_npt; options map to its flags (chunk_steps -> --chunk-steps).  Returns
    (json line, molecules, boxes [K+1,3,3], positions [K+1,N,3])."""
    from oracle import omm
    if not os.path.exists(RUN_NPT):
        raise FileNotFoundError(RUN_NPT)
    os.makedirs(workdir, exist_ok=True)
    xml, pos, out = (os.path.join(workdir, f) for f in ("system.xml", "positions.f64", "out.bin"))
    sim = omm.Simulation(desc, "Reference", pme=pme)
    if omm.lib().omm_system_serialize(sim.sys, xml.encode()) != 0:
        raise RuntimeError("System serialization failed")
    sim.close()
    np.ascontiguousarray(desc.positions, dtype="<f8").tofile(pos)
    cmd = [RUN_NPT, xml, pos, out, "--platform", platform, "--plugin", PLUGIN]
    for k, v in options.items():
        cmd += ["--" + k.replace("_", "-"), str(v)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=timeout, cwd=ROOT)
    if r.returncode != 0:
        raise RuntimeError("run_npt failed: " + r.stdout[-2000:] + r.stderr[-2000:])
    line = json.loads(r.stdout.strip().splitlines()[-1])
    raw = open(out, "rb").read()
    nmol = int(np.frombuffer(raw, "<i4", 1)[0])
    start = np.frombuffer(raw, "<i4", nmol + 1, 4)
    off = 4*(nmol + 2)
    atoms = np.frombuffer(raw, "<i4", int(start[-1]), off)
    off += 4*int(start[-1])
    frames = np.frombuffer(raw, "<f8", offset=off).reshape(-1, 3 + desc.natoms, 3)
    mols = [atoms[start[m]:start[m+1]].tolist() for m in range(nmol)]
    return line, mols, frames[:, :3].copy(), frames[:, 3:].copy()
