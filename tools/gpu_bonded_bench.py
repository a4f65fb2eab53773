"""What the RB and CMAP segments of k_bonded cost: DHFR against DHFR-CMAP-RB (one H100), in one process.

DHFR-CMAP-RB is DHFR with its 7,310 periodic torsions written as Ryckaert-Bellemans torsions and the 8 CHARMM36 CMAP maps
(tests/golden/charmm36_cmap.npz) on its 157 backbone phi/psi pairs.  For each system: the bonded phase alone
(b200md_time_phase(6): bonds, angles, torsions, RB, CMAP and exceptions in one k_bonded launch) and the device-timed ns/day of
the step path (Langevin 2 fs, CUDA events on the engine's stream, the two engines alternating A B A B).  The card name, power
limit and max SM clock come from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_bonded_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gpu_mixed_bench import gpu_info, device_timed      # noqa: E402


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    args = ap.parse_args()
    import numpy as np
    import torch
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_bonded_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    z = np.load(os.path.join(ROOT, "tests", "golden", "charmm36_cmap.npz"))
    descs = {"dhfr": d, "dhfr_cmap_rb": systems.with_cmap(systems.periodic_to_rb(d), z["size"], z["energy"], z["coeff"])}
    flush = torch.empty(256*1024*1024, dtype=torch.uint8, device="cuda")
    engines = {}
    for name, desc in descs.items():
        eng = Engine(desc)
        eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7, 1e-5)
        eng.step(300)
        stream = torch.cuda.ExternalStream(eng.stream())
        for _ in range(args.warmup):
            eng.step(args.md_steps)
        engines[name] = (eng, stream)
    ms = {name: [] for name in descs}
    for _ in range(args.rounds):
        for name in descs:
            eng, stream = engines[name]
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
    out = {"gpu": info, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps, "rounds": args.rounds}
    for name, desc in descs.items():
        eng = engines[name][0]
        eng.compute()
        rates = [0.002e-3*86400/(m*1e-3) for m in ms[name]]
        out[name] = {"torsions": len(desc.tor_i), "rb_torsions": len(desc.rb_i), "cmap_terms": len(desc.cmap_map),
                     "ns_per_day": rates, "ns_per_day_best": max(rates), "us_per_step": [1e3*m for m in ms[name]],
                     "bonded_phase_us": 1e3*eng.time_phase("bonded", 200)}
    out["cmap_rb_over_dhfr"] = out["dhfr_cmap_rb"]["ns_per_day_best"]/out["dhfr"]["ns_per_day_best"]
    for eng, _ in engines.values():
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
