"""Single vs mixed precision on DHFR (one H100), in one process.

Device-timed ns/day with the protocol of bench.py (Langevin 2 fs, 300 equilibration steps, warm-up, 500-step bench steps,
CUDA events on the engine's stream), alternating single and mixed engines A B A B so that both see the same machine state;
the integrate phase alone (b200md_time_phase(4)) for each; and the end-to-end rate through the OpenMM plugin
(Context + LangevinMiddleIntegrator::step) with Precision=single and Precision=mixed.  The card name, power limit and max SM
clock come from a read-only nvidia-smi query in the same call.  Prints one JSON line.

    python tools/gpu_mixed_bench.py [--rounds 3] [--steps 10] [--warmup 2] [--md-steps 500]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=60)
    name, power, clock = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def device_timed(eng, torch, stream, flush, steps, md):
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    ev0.record(stream)
    for _ in range(steps):
        with torch.cuda.stream(stream):
            flush.zero_()
        eng.step(md)
    ev1.record(stream)
    torch.cuda.synchronize()
    return ev0.elapsed_time(ev1)/(steps*md)          # ms per MD step


def plugin_rate(d, precision, md):
    """ns/day of LangevinMiddleIntegrator::step(1) x md through the plugin, host clock around a synchronising getState."""
    from oracle import omm
    from openmm_b200 import systems
    sim = omm.Simulation(d, "B200", integrator=(systems.INT_LANGEVIN_MIDDLE, 300.0, 1.0, 0.002), pme=d.pme_parameters(),
                         props="Precision=" + precision)
    assert sim.platform() == "B200"
    sim.step(300)
    sim.state(positions=True)
    t0 = time.perf_counter()
    sim.step(md)
    sim.state(positions=True)
    sec = time.perf_counter() - t0
    sim.close()
    return 0.002e-3*md*86400/sec


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--md-steps", type=int, default=500)
    args = ap.parse_args()
    import torch
    from openmm_b200 import systems, Engine
    if not torch.cuda.is_available():
        raise SystemExit("gpu_mixed_bench.py: no CUDA device")
    info = gpu_info()
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    flush = torch.empty(256*1024*1024, dtype=torch.uint8, device="cuda")
    engines = {}
    for p in ("single", "mixed"):
        eng = Engine(d, precision=p)
        eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7, 1e-5)
        eng.step(300)
        stream = torch.cuda.ExternalStream(eng.stream())
        for _ in range(args.warmup):
            eng.step(args.md_steps)
        engines[p] = (eng, stream)
    ms = {"single": [], "mixed": []}
    for _ in range(args.rounds):
        for p in ("single", "mixed"):
            eng, stream = engines[p]
            ms[p].append(device_timed(eng, torch, stream, flush, args.steps, args.md_steps))
    out = {"gpu": info, "workload": "dhfr", "md_steps_per_bench_step": args.md_steps, "bench_steps": args.steps, "rounds": args.rounds}
    for p in ("single", "mixed"):
        eng = engines[p][0]
        rates = [0.002e-3*86400/(m*1e-3) for m in ms[p]]
        out[p] = {"ns_per_day": rates, "ns_per_day_best": max(rates), "us_per_step": [1e3*m for m in ms[p]],
                  "integrate_phase_us": 1e3*eng.time_phase("integrate", 200)}
    out["mixed_over_single"] = out["mixed"]["ns_per_day_best"]/out["single"]["ns_per_day_best"]
    for eng, _ in engines.values():
        eng.close()
    try:
        from oracle import omm
        plugin = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
        if omm.available() and os.path.exists(plugin):
            omm.load_plugin(plugin)
            out["plugin_e2e_ns_per_day"] = {p: plugin_rate(d, p, args.md_steps) for p in ("single", "mixed")}
    except OSError as e:
        out["plugin_e2e_ns_per_day"] = "not measured: %s" % e
    print(json.dumps(out))


if __name__ == "__main__":
    main()
