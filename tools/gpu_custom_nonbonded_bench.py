"""What CustomNonbondedForce costs (one H100, one process).
- Device-timed ns/day of the step path (CUDA events on the engine's stream) of DHFR (data/dhfr.npz, PME 0.9 nm, HBonds),
  DHFR-LJ-table (its Lennard-Jones moved into a CustomNonbondedForce of Discrete2DFunction tables) and DHFR-NBFIX (overridden
  pairs, switching at 0.8 nm; tests/custom_nonbonded_harness.py), LangevinMiddle 2 fs, alternating round by round.
- The custom nonbonded kernel alone (b200md_time_phase phase 14, k_custom_nonbonded, forces only) and the tile kernel alone
  (phase 0), on DHFR-LJ-table.
- The plugin path: host clock around --plugin-steps steps ending in a state read, the three Systems alternating.
The card name, power limit and max SM clock come from a read-only nvidia-smi query in the same call.  Prints one JSON line with
the arguments used.

    python tools/gpu_custom_nonbonded_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500] [--plugin-steps 1000]
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

DT, FRICTION, TEMPERATURE = 0.002, 1.0, 300.0


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    ap.add_argument("--phase-reps", type=int, default=200)
    ap.add_argument("--plugin-steps", type=int, default=1000)
    args = ap.parse_args()
    import torch
    import custom_nonbonded_harness as H
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_custom_nonbonded_bench.py: no CUDA device")
    info = gpu_info()
    plain = systems.SystemDesc.load(H.DHFR).rounded()
    configs = {"dhfr": plain, "dhfr_lj_table": H.engine_desc(False), "dhfr_nbfix": H.engine_desc(True)}
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
    phases = {"custom_nonbonded_kernel_us": [], "tile_kernel_us": []}
    for _ in range(args.rounds):
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
        eng = steppers["dhfr_lj_table"][0]
        for phase, label in (("custom_nonbonded", "custom_nonbonded_kernel_us"), ("pair", "tile_kernel_us")):
            eng.time_phase(phase, 20)
            phases[label].append(1e3*eng.time_phase(phase, args.phase_reps))
    for eng, _ in steppers.values():
        eng.close()
    # the plugin path
    H.omm.load_plugin(os.path.join(ROOT, "plugin", "libOpenMMB200.so"))
    table, f = H.dhfr_lj_table()
    nbfix, g = H.dhfr_lj_table(nbfix=True)
    integ = (systems.INT_LANGEVIN_MIDDLE, TEMPERATURE, FRICTION, DT)
    sims = {"dhfr": H.Simulation(plain, "B200", integrator=integ, pme=plain.pme_parameters()),
            "dhfr_lj_table": H.Simulation(table, "B200", forces=[f], integrator=integ, pme=table.pme_parameters()),
            "dhfr_nbfix": H.Simulation(nbfix, "B200", forces=[g], integrator=integ, pme=nbfix.pme_parameters())}
    for s in sims.values():
        s.step(200)
        s.state(energy=True)
    plugin = {k: [] for k in sims}
    for _ in range(args.rounds):
        for k, s in sims.items():
            t = time.perf_counter()
            s.step(args.plugin_steps)
            s.state(energy=True)
            plugin[k].append(DT*1e-3*args.plugin_steps*86400/(time.perf_counter() - t))
    out = {"gpu": info, "args": vars(args), "atoms": plain.natoms, "dt_ps": DT}
    out.update(phases)
    for name in steppers:
        out[name] = {"ns_per_day": [DT*1e-3*86400/(m*1e-3) for m in ms[name]], "us_per_step": [1e3*m for m in ms[name]],
                     "plugin_ns_per_day": plugin[name]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
