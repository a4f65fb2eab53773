"""What custom angles and custom compound bonds cost (k_custom and k_compound, one H100, one process).

- Device-timed ns/day of the step path (LangevinMiddle 2 fs, CUDA events on the engine's stream), the variants alternating
  round by round: DHFR; DHFR plus one six-particle orientational restraint (systems.with_orientational_restraint: one
  distance, two angles, three dihedrals, 19 programs); DHFR with its harmonic angles as custom angles
  (systems.angles_to_custom); DHFR with its angles and its 7,310 periodic torsions as compound bonds (angles_to_compound,
  torsions_to_compound: up to 13 programs per term).  The last is a stress case that characterises the interpreter, not a way
  anybody would write a force field.
- The bonded kernels alone (b200md_time_phase): k_bonded of DHFR (phase 6), k_custom of the custom-angle variant (phase 7),
  k_compound of the restraint and of the stress case (phase 8).
The programs come from the plugin's translator (tests/custom_harness.py).  The card name, power limit and max SM clock
come from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_custom_compound_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_mixed_bench import gpu_info, device_timed      # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    ap.add_argument("--phase-reps", type=int, default=500)
    args = ap.parse_args()
    import torch
    import custom_harness as harness
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_custom_compound_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    configs = {"dhfr": d, "dhfr_restraint": systems.with_orientational_restraint(d, systems.restraint_atoms(d)),
               "dhfr_custom_angles": systems.angles_to_custom(d),
               "dhfr_all_compound": systems.torsions_to_compound(systems.angles_to_compound(d))}
    phases = {"dhfr": ("bonded", "k_bonded_us"), "dhfr_restraint": ("custom_compound", "k_compound_restraint_us"),
              "dhfr_custom_angles": ("custom_torsions", "k_custom_angles_us"),
              "dhfr_all_compound": ("custom_compound", "k_compound_all_us")}
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
    ms = {name: [] for name in steppers}
    kernel = {label: [] for _, label in phases.values()}
    for _ in range(args.rounds):
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
        for name, (eng, _) in steppers.items():
            phase, label = phases[name]
            eng.time_phase(phase, 20)
            kernel[label].append(1e3*eng.time_phase(phase, args.phase_reps))
    out = {"gpu": info, "rounds": args.rounds, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps,
           "angles": len(d.angle_i), "torsions": len(d.tor_i)}
    out.update(kernel)
    for name in steppers:
        rates = [0.002e-3*86400/(m*1e-3) for m in ms[name]]
        out[name] = {"ns_per_day": rates, "us_per_step": [1e3*m for m in ms[name]]}
    for eng, _ in steppers.values():
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
