"""What generalized Born costs (GBSAOBCForce, OBC II + ACE; one H100, one process).

- Device-timed ns/day of the step path (CUDA events on the engine's stream) on DHFR-GBSA with the reference benchmark's
  implicit-solvent protocol (tests/golden/dhfr_gbsa.npz: amber99sb + amber99_obc, CutoffNonPeriodic 2 nm, HBonds;
  LangevinMiddle 4 fs, 91/ps), alternating round by round with the same System without its GBSAOBCForce.
- The GB chain alone (b200md_time_phase phase 10: k_gb_born, k_gb_radii, k_gb_pairs, k_gb_fold, k_gb_chain) and the tile
  kernel alone (phase 0), to set the chain's length beside the kernel it runs beside.
- The baseline leg: the reference's CPU platform (oracle/_ref/libOpenMMCPU.so) on the same host, same System and protocol,
  wall-clock ns/day over --cpu-steps steps.
The card name, power limit and max SM clock come from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_gbsa_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500] [--cpu-steps 200]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_mixed_bench import gpu_info, device_timed      # noqa: E402

DT, FRICTION, TEMPERATURE = 0.004, 91.0, 300.0


def cpu_leg(d, steps):
    """ns/day of the reference's CPU platform on this host (None when the library is not there)"""
    import gbsa_harness as H
    from openmm_b200 import systems
    path = os.path.join(ROOT, "oracle", "_ref", "libOpenMMCPU.so")
    if not (H.available() and os.path.exists(path)):
        return None
    H.omm.load_plugin(path)
    sim = H.Simulation(d, "CPU", integrator=(systems.INT_LANGEVIN_MIDDLE, TEMPERATURE, FRICTION, DT))
    sim.step(20)
    t0 = time.perf_counter()
    sim.step(steps)
    sim.state(energy=True)
    sec = time.perf_counter() - t0
    sim.close()
    return DT*1e-3*steps*86400/sec


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    ap.add_argument("--phase-reps", type=int, default=500)
    ap.add_argument("--cpu-steps", type=int, default=200)
    args = ap.parse_args()
    import torch
    import gbsa_harness as H
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_gbsa_bench.py: no CUDA device")
    info = gpu_info()
    d = H.dhfr_gbsa().rounded()
    configs = {"dhfr_gbsa": d, "dhfr_gbsa_without_gb": H.without_gbsa(d)}
    flush = torch.empty(256*1024*1024, dtype=torch.uint8, device="cuda")
    steppers = {}
    for name, desc in configs.items():
        eng = Engine(desc)
        eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, DT, TEMPERATURE, FRICTION, 7, 1e-5)
        eng.step(300)
        stream = torch.cuda.ExternalStream(eng.stream())
        for _ in range(args.warmup):
            eng.step(args.md_steps)
        steppers[name] = (eng, stream)
    ms = {name: [] for name in steppers}
    phases = {"gb_chain_us": [], "tile_kernel_us": []}
    for _ in range(args.rounds):
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
        eng = steppers["dhfr_gbsa"][0]
        for phase, label in (("gbsa", "gb_chain_us"), ("pair", "tile_kernel_us")):
            eng.time_phase(phase, 20)
            phases[label].append(1e3*eng.time_phase(phase, args.phase_reps))
    out = {"gpu": info, "rounds": args.rounds, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps,
           "atoms": d.natoms, "dt_ps": DT}
    out.update(phases)
    for name in steppers:
        out[name] = {"ns_per_day": [DT*1e-3*86400/(m*1e-3) for m in ms[name]], "us_per_step": [1e3*m for m in ms[name]]}
    for eng, _ in steppers.values():
        eng.close()
    out["reference_cpu_ns_per_day"] = cpu_leg(d, args.cpu_steps)
    out["host_cpus"] = os.cpu_count()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
