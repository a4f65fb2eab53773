"""One-shot iteration script: parity error summary on the real systems + step timing for a workload."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from openmm_b200 import systems, Engine
from openmm_b200.engine import TERM_NB_DIRECT, TERM_NB_RECIP, TERM_ALL

mode = sys.argv[1]
names = sys.argv[2:] or ["dhfr"]
for name in names:
    if os.path.exists(os.path.join("data", name + ".npz")):
        d = systems.SystemDesc.load(os.path.join("data", name + ".npz")).rounded()
    else:
        import bench
        d = bench.load_workload(name)
    eng = Engine(d)
    if mode == "parity":
        from oracle import omm
        sim = omm.Simulation(d, "Reference", pme=d.pme_parameters(), recip_group=1)
        for label, terms, groups in (("recip", TERM_NB_RECIP, 2), ("direct+bonded", TERM_ALL & ~TERM_NB_RECIP, 1), ("all", TERM_ALL, 3)):
            e = eng.compute(terms); f = eng.get_forces()
            fr, er = sim.forces_energy(groups)
            err = np.abs(f - fr).max(axis=1)
            rel = err/np.maximum(1, np.linalg.norm(fr, axis=1))
            print("%s %-14s E %.4f ref %.4f | max rel %.3e abs %.3e | n(rel>1e-4)=%d n(>5e-5)=%d" % (name, label, e, er, rel.max(), err.max(), (rel > 1e-4).sum(), (rel > 5e-5).sum()), flush=True)
    else:
        eng.set_integrator(systems.INT_LANGEVIN, 0.002, 300.0, 1.0, 7, 1e-5)
        stream = torch.cuda.ExternalStream(eng.stream())
        nst = 2000 if d.natoms < 200000 else 200
        eng.step(nst//2); eng.synchronize()
        best = 1e9
        for rep in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream); eng.step(nst); e1.record(stream); torch.cuda.synchronize()
            best = min(best, 1e3*e0.elapsed_time(e1)/nst)
        st = eng.stats()
        ph = {k: round(1e3*eng.time_phase(k, 20), 2) for k in ["pair", "pme_spread", "pme_fft_conv", "pme_gather", "bonded", "integrate", "list_build"]} if mode == "timeph" else {}
        print("%s %.1f us/step %.1f ns/day builds %d tiles %d %s env PAD=%s" % (name, best, 172800.0/best, st.get("list_builds", -1), st.get("num_tiles", -1), ph,
              os.environ.get("B200MD_PAD_FRACTION")), flush=True)
