"""What custom torsions cost (k_custom_torsion, one H100, one process).

- The bonded phase (b200md_time_phase 6: k_bonded, and k_custom_torsion behind it when there are custom torsions) and
  k_custom_torsion alone (phase 7), on DHFR and on DHFR with its 7,310 periodic torsions written as the CustomTorsionForce
  k*(1+cos(n*theta-theta0)) (systems.periodic_to_custom).
- Device-timed ns/day of the step path (LangevinMiddle 2 fs, CUDA events on the engine's stream) for DHFR against
  DHFR-CHARMM: DHFR plus the CHARMM36 CMAP maps on its backbone and CharmmPsfFile-form impropers (systems.with_cmap,
  systems.with_charmm_impropers).
The configurations alternate for --rounds rounds.  The programs come from the plugin's translator (tests/
custom_torsion_harness.py over oracle/_ref/tests/libcustom_torsion_capi.so).  The card name, power limit and max SM clock come
from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_custom_torsion_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500]
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
    ap.add_argument("--phase-reps", type=int, default=200)
    args = ap.parse_args()
    import numpy as np
    import torch
    import custom_torsion_harness as harness
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_custom_torsion_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    z = np.load(os.path.join(ROOT, "tests", "golden", "charmm36_cmap.npz"))
    charmm = harness.compiled(systems.with_cmap(systems.with_charmm_impropers(d), z["size"], z["energy"], z["coeff"]))
    custom = harness.compiled(systems.periodic_to_custom(d))
    engines = {name: Engine(desc) for name, desc in (("dhfr", d), ("dhfr_custom_periodic", custom))}
    phases = {name: {"bonded_us": [], "custom_torsion_us": []} for name in engines}
    for _ in range(args.rounds):
        for name, eng in engines.items():
            eng.compute()
            phases[name]["bonded_us"].append(1e3*eng.time_phase("bonded", args.phase_reps))
            if name != "dhfr":
                phases[name]["custom_torsion_us"].append(1e3*eng.time_phase("custom_torsions", args.phase_reps))
    for eng in engines.values():
        eng.close()
    flush = torch.empty(256*1024*1024, dtype=torch.uint8, device="cuda")
    steppers = {}
    for name, desc in (("dhfr", d), ("dhfr_charmm", charmm)):
        eng = Engine(desc)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 7, 1e-5)
        eng.step(300)
        stream = torch.cuda.ExternalStream(eng.stream())
        for _ in range(args.warmup):
            eng.step(args.md_steps)
        steppers[name] = (eng, stream)
    ms = {name: [] for name in steppers}
    for _ in range(args.rounds):
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
    out = {"gpu": info, "rounds": args.rounds, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps,
           "phases": phases, "custom_periodic_torsions": len(custom.custom_prog),
           "dhfr_charmm": {"impropers": len(charmm.custom_prog), "cmap_terms": len(charmm.cmap_map)}}
    for name in steppers:
        rates = [0.002e-3*86400/(m*1e-3) for m in ms[name]]
        out.setdefault(name, {}).update({"ns_per_day": rates, "us_per_step": [1e3*m for m in ms[name]]})
    for eng, _ in steppers.values():
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
