"""What an RMSDForce and a CustomCVForce cost (one H100, one process, every variant alternating round by round).

- Engine, device-timed ns/day of the step path (LangevinMiddle 2 fs, CUDA events on the engine's stream): DHFR; DHFR plus a bare
  RMSDForce over its 1,268 solute heavy atoms (systems.solute_heavy_atoms), inside the captured step graph with no host sync.
- The three RMSD kernels alone (b200md_time_phase phase 13).
- Through the plugin (Context + LangevinMiddleIntegrator.step, host clock around steps that end in a state read): DHFR, and DHFR
  with the RMSD restraint 0.5 k max(0, rmsd - r0)^2 as a CustomCVForce.  A CustomCVForce step evaluates its variable in the
  inner context and reads its value back: one host sync per variable per step, as on the reference's GPU platforms.
The card name, power limit and max SM clock come from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_custom_cv_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500] [--plugin-steps 2000]
"""
import argparse
import copy
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_mixed_bench import gpu_info, device_timed      # noqa: E402


def with_rmsd(d, atoms, seed=1):
    """d plus one RMSDForce over `atoms`, its reference positions 0.05 nm (per coordinate, normal) from d's"""
    out = copy.copy(d)
    ref = np.asarray(d.positions, dtype=np.float64)[atoms] + np.random.default_rng(seed).normal(0.0, 0.05, (len(atoms), 3))
    out.rmsd_start, out.rmsd_atoms = np.array([0, len(atoms)], np.int32), np.asarray(atoms, np.int32)
    out.rmsd_ref, out.rmsd_group = ref, np.zeros(1, np.int32)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    ap.add_argument("--phase-reps", type=int, default=500)
    ap.add_argument("--plugin-steps", type=int, default=2000)
    args = ap.parse_args()
    import torch
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_custom_cv_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    atoms = systems.solute_heavy_atoms(d)
    configs = {"dhfr": d, "dhfr_rmsd": with_rmsd(d, atoms)}
    flush = torch.empty(256*1024*1024, dtype=torch.uint8, device="cuda")
    steppers = {}
    for name, desc in configs.items():
        eng = Engine(desc)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7, 1e-5)
        eng.step(300)
        stream = torch.cuda.ExternalStream(eng.stream())
        for _ in range(args.warmup):
            eng.step(args.md_steps)
        steppers[name] = (eng, stream)
    import time
    import rmsd_harness as H
    H.omm.load_plugin(os.path.join(ROOT, "plugin", "libOpenMMB200.so"))
    ref = np.array(d.positions, dtype=np.float64)
    ref[atoms] += np.random.default_rng(1).normal(0.0, 0.05, (len(atoms), 3))
    cv = {"energy": "0.5*k*max(0, rmsd-r0)^2", "variables": [("rmsd", "rmsd", atoms, ref)], "globals": [("k", 5000.0, False), ("r0", 0.02, False)]}
    integ = (systems.INT_LANGEVIN_MIDDLE, 300.0, 1.0, 0.002)
    sims = {"plugin_dhfr": H.Simulation(d, "B200", pme=d.pme_parameters(), integrator=integ),
            "plugin_dhfr_cv_rmsd_restraint": H.CVSimulation(d, "B200", cv=cv, pme=d.pme_parameters(), integrator=integ)}
    for s in sims.values():
        s.set_velocities_to_temperature(300.0, 3)
        s.step(200)
        s.state(energy=True)
    plugin_ms = {name: [] for name in sims}
    ms = {name: [] for name in steppers}
    kernels = []
    for _ in range(args.rounds):
        for name, s in sims.items():
            t0 = time.perf_counter()
            s.step(args.plugin_steps)
            s.state(positions=True)
            plugin_ms[name].append(1e3*(time.perf_counter() - t0)/args.plugin_steps)
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
        eng = steppers["dhfr_rmsd"][0]
        eng.time_phase("rmsd", 20)
        kernels.append(1e3*eng.time_phase("rmsd", args.phase_reps))
    out = {"gpu": info, "rounds": args.rounds, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps,
           "rmsd_atoms": int(len(atoms)), "rmsd_kernels_us": kernels}
    for name in steppers:
        out[name] = {"ns_per_day": [0.002e-3*86400/(m*1e-3) for m in ms[name]], "us_per_step": [1e3*m for m in ms[name]]}
    for name in sims:
        out[name] = {"ns_per_day": [0.002e-3*86400/(m*1e-3) for m in plugin_ms[name]], "us_per_step": [1e3*m for m in plugin_ms[name]]}
    for eng, _ in steppers.values():
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
