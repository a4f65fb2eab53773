"""What custom centroid bonds cost (k_centroid_centers, k_compound at the centres, k_centroid_scatter; one H100, one process).

- Device-timed ns/day of the step path (LangevinMiddle 2 fs, CUDA events on the engine's stream), the variants alternating
  round by round: DHFR; DHFR plus a mass-weighted centre-of-mass distance restraint between the two halves of its solute heavy
  atoms (systems.solute_halves, two groups of about 630 atoms); DHFR plus one centre-of-mass position restraint per water
  (about 7,000 three-atom groups, one bond each), a stress case.
- The three centroid kernels alone (b200md_time_phase phase 9) for both restraints, and k_compound alone (phase 8) for DHFR
  with the six-particle orientational restraint, to set beside the same figure of the parent's tools/gpu_custom_compound_bench.py.
The programs come from the plugin's translator (tests/centroid_harness.py).  The card name, power limit and max SM clock come
from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_custom_centroid_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_mixed_bench import gpu_info, device_timed      # noqa: E402


def water_restraints(d):
    """DHFR plus one harmonic restraint of every water's centre of mass to where it is now, shifted by 0.01 nm"""
    from openmm_b200 import systems
    waters = [m for m in d.molecules() if len(m) == 3]
    x, m = np.asarray(d.positions), np.asarray(d.masses)
    centres = np.array([m[w] @ x[w]/m[w].sum() for w in waters]) + 0.01
    params = np.concatenate([np.full((len(waters), 1), 1000.0), centres], axis=1)
    return systems.with_centroid_restraint(d, waters, "0.5*k*((x1-x0)^2+(y1-y0)^2+(z1-z0)^2)", params, ("k", "x0", "y0", "z0"),
                                           bonds=np.arange(len(waters)).reshape(-1, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    ap.add_argument("--phase-reps", type=int, default=500)
    args = ap.parse_args()
    import torch
    import centroid_harness as harness
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_custom_centroid_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    a, b = systems.solute_halves(d)
    configs = {"dhfr": d,
               "dhfr_com_distance": systems.with_centroid_restraint(d, [a, b], systems.COM_DISTANCE_RESTRAINT, [[2000.0, 1.0]], ("k", "r0")),
               "dhfr_water_restraints": water_restraints(d)}
    phases = {"dhfr_com_distance": [("custom_centroid", "centroid_com_distance_us")],
              "dhfr_water_restraints": [("custom_centroid", "centroid_water_restraints_us")]}
    flush = torch.empty(256*1024*1024, dtype=torch.uint8, device="cuda")
    steppers = {}
    for name, desc in configs.items():
        eng = Engine(harness.compiled(desc))
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7, 1e-5)
        eng.step(300)
        stream = torch.cuda.ExternalStream(eng.stream())
        for _ in range(args.warmup):
            eng.step(args.md_steps)
        steppers[name] = (eng, stream)
    orient = Engine(harness.compiled(systems.with_orientational_restraint(d, systems.restraint_atoms(d))))
    ms = {name: [] for name in steppers}
    kernel = {label: [] for v in phases.values() for _, label in v}
    kernel["k_compound_restraint_us"] = []
    for _ in range(args.rounds):
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
        for name, (eng, _) in steppers.items():
            for phase, label in phases.get(name, ()):
                eng.time_phase(phase, 20)
                kernel[label].append(1e3*eng.time_phase(phase, args.phase_reps))
        orient.time_phase("custom_compound", 20)
        kernel["k_compound_restraint_us"].append(1e3*orient.time_phase("custom_compound", args.phase_reps))
    out = {"gpu": info, "rounds": args.rounds, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps,
           "half_groups": [len(a), len(b)], "water_groups": len(configs["dhfr_water_restraints"].ccentroid_expr)}
    out.update(kernel)
    for name in steppers:
        rates = [0.002e-3*86400/(m*1e-3) for m in ms[name]]
        out[name] = {"ns_per_day": rates, "us_per_step": [1e3*m for m in ms[name]]}
    for eng, _ in steppers.values():
        eng.close()
    orient.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
