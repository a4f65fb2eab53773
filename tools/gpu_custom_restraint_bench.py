"""What custom bonds and externals cost (k_custom, one H100, one process per measurement of another build).

- k_custom alone (b200md_time_phase 7) on DHFR with its 7,310 periodic torsions written as the CustomTorsionForce
  k*(1+cos(n*theta-theta0)) (systems.periodic_to_custom): this build, and, with --parent DIR, the build in the source tree DIR
  (its own openmm_b200 package and libb200md.so, run in a subprocess with the same compiled programs), alternating round by
  round.  The kernel now serves three classes; this is what the torsions pay for it.
- Device-timed ns/day of the step path (LangevinMiddle 2 fs, CUDA events on the engine's stream) for DHFR, DHFR plus
  position restraints on its 1,268 solute heavy atoms (k*periodicdistance(x, y, z, x0, y0, z0)^2), DHFR-CHARMM (DHFR plus the
  CHARMM36 CMAP maps and CharmmPsfFile-form impropers) and DHFR-CHARMM plus the same restraints, alternating.
The programs come from the plugin's translator (tests/custom_harness.py).  The card name, power limit and max SM clock
come from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_custom_restraint_bench.py [--parent DIR] [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from gpu_mixed_bench import gpu_info, device_timed      # noqa: E402

# phase 7 of DHFR with custom periodic torsions, in a tree given as argv[1], with the programs of the npz argv[2]: one float (us)
PHASE7_CHILD = """
import sys, os, json
import numpy as np
sys.path.insert(0, sys.argv[1])
from openmm_b200 import systems, Engine
d = systems.SystemDesc.load(os.path.join(sys.argv[1], "data", "dhfr.npz")).rounded()
c = systems.periodic_to_custom(d)
z = np.load(sys.argv[2])
c.custom_prog_start, c.custom_op, c.custom_arg, c.custom_imm = z["start"], z["op"], z["arg"], z["imm"]
eng = Engine(c)
eng.compute()
eng.time_phase("custom_torsions", 20)
print(json.dumps(1e3*eng.time_phase("custom_torsions", int(sys.argv[3]))))
"""


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--parent", default=None, help="a source tree with a built libb200md.so to compare phase 7 against")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    ap.add_argument("--phase-reps", type=int, default=500)
    args = ap.parse_args()
    import numpy as np
    import torch
    import custom_harness as harness
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_custom_restraint_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    custom = harness.compiled(systems.periodic_to_custom(d))
    programs = os.path.join(tempfile.mkdtemp(), "programs.npz")
    np.savez(programs, start=custom.custom_prog_start, op=custom.custom_op, arg=custom.custom_arg, imm=custom.custom_imm)
    trees = {"this": ROOT}
    if args.parent:
        trees["parent"] = os.path.abspath(args.parent)
    phase7 = {name: [] for name in trees}
    for _ in range(args.rounds):
        for name, tree in trees.items():
            p = subprocess.run([sys.executable, "-c", PHASE7_CHILD, tree, programs, str(args.phase_reps)], capture_output=True, text=True,
                               env=dict(os.environ, B200MD_LIB=os.path.join(tree, "openmm_b200", "libb200md.so")))
            if p.returncode != 0:
                raise SystemExit("phase 7 of %s failed: %s" % (tree, p.stderr[-2000:]))
            phase7[name].append(float(p.stdout.strip().splitlines()[-1]))
    z = np.load(os.path.join(ROOT, "tests", "golden", "charmm36_cmap.npz"))
    charmm = systems.with_cmap(systems.with_charmm_impropers(d), z["size"], z["energy"], z["coeff"])
    atoms = systems.solute_heavy_atoms(d)
    configs = {"dhfr": d, "dhfr_restrained": systems.with_position_restraints(d, atoms, 400.0),
               "dhfr_charmm": charmm, "dhfr_charmm_restrained": systems.with_position_restraints(charmm, atoms, 400.0)}
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
    for _ in range(args.rounds):
        for name, (eng, stream) in steppers.items():
            ms[name].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
    out = {"gpu": info, "rounds": args.rounds, "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps,
           "phase7_custom_periodic_us": phase7, "custom_periodic_torsions": len(custom.custom_prog), "restraints": len(atoms)}
    for name in steppers:
        rates = [0.002e-3*86400/(m*1e-3) for m in ms[name]]
        out[name] = {"ns_per_day": rates, "us_per_step": [1e3*m for m in ms[name]]}
    for eng, _ in steppers.values():
        eng.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
