"""GPU tests of RBTorsionForce and CMAPTorsionForce on the platform (the RB and CMAP segments of k_bonded): the reference's own
test bodies, the C-ABI against the live Reference platform on DHFR-CMAP-RB (DHFR with its torsions in Ryckaert-Bellemans form
and the CHARMM36 maps on its 157 backbone phi/psi pairs), force groups, periodic terms, parameter updates, the molecule wrap,
the plugin's step paths and the multi-GPU force decomposition."""
import os
import subprocess
import sys
import numpy as np
import pytest
from conftest import relative_force_error, ROOT, GOLDEN

pytestmark = pytest.mark.gpu
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")
REFTESTS = os.path.join(ROOT, "oracle", "_ref", "tests")


@pytest.fixture(scope="module")
def harness():
    """Reference-side RB and CMAP forces (tests/cmap_rb_harness.py), with the plugin loaded"""
    import cmap_rb_harness
    if not cmap_rb_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where /root/reference exists")
    cmap_rb_harness.omm.load_plugin(PLUGIN)
    return cmap_rb_harness


def _maps():
    z = np.load(os.path.join(GOLDEN, "charmm36_cmap.npz"))
    return z["size"], z["energy"], z["coeff"]


def dhfr_cmap_rb(rb=True):
    """DHFR-CMAP-RB (rb=False: the same with its periodic torsions), fp32-representable positions."""
    from openmm_b200 import systems
    d = systems.SystemDesc.load(os.path.join(ROOT, "data", "dhfr.npz")).rounded()
    return systems.with_cmap(systems.periodic_to_rb(d) if rb else d, *_maps())


@pytest.fixture(scope="module")
def dhfr():
    return dhfr_cmap_rb()


# ---------------------------------------------------------------------------------------------------- reference test bodies
@pytest.mark.parametrize("name", ["TestB200RBTorsionForce", "TestB200CMAPTorsionForce", "TestB200MixedRBTorsionForce",
                                  "TestB200MixedCMAPTorsionForce"])
def test_reference_own_test_bodies_pass(name):
    exe = os.path.join(REFTESTS, name)
    if not os.path.exists(exe):
        pytest.fail("%s not built (make -C plugin reftests where /root/reference exists)" % exe)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=dict(os.environ, B200_PLUGIN=PLUGIN))
    assert p.returncode == 0 and "Done" in p.stdout, p.stdout[-2000:] + p.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------- C-ABI against Reference
def _group_close(f, e, fr, er):
    """one group alone: both sides are double, only the 2^-32 fixed-point force resolution differs"""
    assert np.abs(f - fr).max() <= 1e-6*np.abs(fr).max()
    assert abs(e - er) <= 1e-8*abs(er)


def test_dhfr_cmap_rb_matches_reference_platform(harness, dhfr):
    from openmm_b200 import Engine, engine
    pme = dhfr.pme_parameters()
    ref = harness.Simulation(dhfr, "Reference", pme=pme, force_groups={"rb_torsions": 3, "cmap": 4})
    eng = Engine(dhfr)
    e = eng.compute()
    f = eng.get_forces()
    fr, er = ref.forces_energy()
    assert relative_force_error(f, fr) < 1e-4 and abs(e - er)/abs(er) < 1e-4
    for term, group in ((engine.TERM_RB_TORSIONS, 3), (engine.TERM_CMAP, 4)):
        e = eng.compute(term)
        fr, er = ref.forces_energy(1 << group)
        _group_close(eng.get_forces(), e, fr, er)


def test_rb_torsions_equal_periodic_torsions_on_the_engine(dhfr):
    from openmm_b200 import Engine, engine
    per = Engine(dhfr_cmap_rb(rb=False))
    ep = per.compute(engine.TERM_TORSIONS)
    fp = per.get_forces()
    rb = Engine(dhfr)
    er = rb.compute(engine.TERM_RB_TORSIONS)
    _group_close(rb.get_forces(), er, fp, ep)


def test_force_groups_match_reference_platform(harness, dhfr):
    from openmm_b200 import Engine, engine
    pme = dhfr.pme_parameters()
    ref = harness.Simulation(dhfr, "Reference", pme=pme, force_groups={"rb_torsions": 3, "cmap": 4})
    eng = Engine(dhfr, bonded_groups={"rb_torsions": np.full(len(dhfr.rb_i), 3), "cmap": np.full(len(dhfr.cmap_map), 4)})
    bonded = engine.TERM_BONDS | engine.TERM_ANGLES | engine.TERM_TORSIONS | engine.TERM_RB_TORSIONS | engine.TERM_CMAP
    for mask in (1 << 3, 1 << 4, (1 << 3) | (1 << 4), 1, 1 | (1 << 4), 0xffffffff):
        # the NonbondedForce and the other bonded forces sit in group 0
        terms = bonded | (engine.TERM_NB_DIRECT | engine.TERM_NB_RECIP if mask & 1 else 0)
        e = eng.compute_groups(terms, mask)
        f = eng.get_forces()
        fr, er = ref.forces_energy(mask)
        if mask & 1:
            assert relative_force_error(f, fr) < 1e-4 and abs(e - er)/abs(er) < 1e-4, mask
        else:
            _group_close(f, e, fr, er)


def _chain(n, box, rng, start):
    """n atoms of a random chain with 0.15 nm steps and tetrahedral-like angles, from start"""
    x = [np.asarray(start, float)]
    d = np.array([1.0, 0.0, 0.0])
    for _ in range(n - 1):
        while True:
            v = rng.standard_normal(3)
            v /= np.linalg.norm(v)
            if -0.6 < v @ d < 0.2:
                break
        d = v
        x.append(x[-1] + 0.15*d)
    return np.array(x)


def _bare(natoms, positions, box, method):
    """natoms uncharged particles without LJ: only the bonded terms act"""
    from openmm_b200 import systems
    z = np.zeros(natoms)
    return systems.SystemDesc(masses=np.full(natoms, 12.0), charges=z, sigmas=np.full(natoms, 0.3), epsilons=z.copy(),
                              positions=positions, box=box, method=method, cutoff=1.0, use_dispersion=False)


def _with_terms(d, n_rb, size, energy, coeff, rng):
    """RB torsions on consecutive quadruples and CMAP terms on consecutive quintuples of d's atoms"""
    d.rb_i, d.rb_j, d.rb_k, d.rb_l = (np.arange(n_rb, dtype=np.int32) + k for k in range(4))
    d.rb_c = rng.uniform(-5, 5, (n_rb, 6))
    m = d.natoms - 4
    d.cmap_atoms = np.array([[i, i+1, i+2, i+3, i+1, i+2, i+3, i+4] for i in range(m)], dtype=np.int32)
    d.cmap_size, d.cmap_energy, d.cmap_coeff = size, energy, coeff.reshape(-1, 16)
    d.cmap_map = (np.arange(m) % len(size)).astype(np.int32)
    return d


def test_periodic_terms_straddling_a_triclinic_box(harness):
    from openmm_b200 import Engine, systems
    rng = np.random.default_rng(11)
    # box vectors exact in fp32, as the positions: both platforms then take the same minimum images
    box = np.array([[2.5, 0.0, 0.0], [0.625, 2.375, 0.0], [-0.5, 0.75, 2.625]])
    x = _chain(40, box, rng, start=(2.3, 2.2, 2.4))
    # every atom wrapped into the box on its own: the chain crosses the faces, only minimum images make it whole
    for k in (2, 1, 0):
        x -= np.floor(x[:, k:k+1]/box[k, k])*box[k]
    x = x.astype(np.float32).astype(np.float64)
    d = _with_terms(_bare(40, x, box, systems.NB_CUTOFF_PERIODIC), 37, *_maps(), rng)
    ref = harness.Simulation(d, "Reference", bonded_periodic=True)
    eng = Engine(d, bonded_groups={"rb_torsions": np.full(37, 0x80), "cmap": np.full(36, 0x80)})
    e = eng.compute()
    fr, er = ref.forces_energy()
    _group_close(eng.get_forces(), e, fr, er)


def test_parameter_updates_match_a_fresh_reference_context(harness):
    from openmm_b200 import Engine, EngineError, systems
    rng = np.random.default_rng(5)
    size, energy, coeff = _maps()
    x = _chain(24, None, rng, start=(1.0, 1.0, 1.0)).astype(np.float32).astype(np.float64)
    d = _with_terms(_bare(24, x, None, systems.NB_NOCUTOFF), 21, size[:3], energy[:3*576], coeff[:3*576], rng)
    eng = Engine(d)
    eng.compute()
    d.rb_c = rng.uniform(-5, 5, (21, 6))
    d.cmap_energy = d.cmap_energy[::-1].copy()*1.5
    d.cmap_coeff = np.concatenate([harness.coefficients(24, d.cmap_energy[576*m:576*(m+1)]) for m in range(3)])
    d.cmap_map = ((np.arange(len(d.cmap_map)) + 1) % 3).astype(np.int32)
    eng.update_rb_torsion_params(d.rb_c)
    eng.update_cmap_params(d.cmap_size, d.cmap_coeff, d.cmap_map)
    e = eng.compute()
    fr, er = harness.Simulation(d, "Reference").forces_energy()
    _group_close(eng.get_forces(), e, fr, er)
    with pytest.raises(EngineError, match="number of maps"):
        eng.update_cmap_params(d.cmap_size[:2], d.cmap_coeff[:2*576], d.cmap_map)
    with pytest.raises(EngineError, match="size of a map"):
        eng.update_cmap_params([24, 24, 12], d.cmap_coeff[:2*576 + 144], d.cmap_map)
    with pytest.raises(EngineError, match="number of CMAP torsions"):
        eng.update_cmap_params(d.cmap_size, d.cmap_coeff, d.cmap_map[:-1])
    with pytest.raises(EngineError, match="map index"):
        eng.update_cmap_params(d.cmap_size, d.cmap_coeff, np.full(len(d.cmap_map), 3))
    with pytest.raises(EngineError, match="number of torsions"):
        eng.update_rb_torsion_params(d.rb_c[:-1])


def test_wrap_keeps_cmap_molecules_whole(harness):
    """A 5-atom CMAP chain without bonds in a PME water box, its first atom put just past two box lengths from the primary
    cell and the others just short of it: the wrap at the list build moves the chain's molecule by whole lattice vectors,
    all five atoms together, only if the CMAP term joins them into one molecule."""
    from openmm_b200 import Engine, systems
    w = systems.water_box(6, cutoff=0.9).rounded()
    L = float(w.box[0][0])
    lo = w.positions.min(axis=0)
    rng = np.random.default_rng(2)
    while True:
        c = _chain(5, None, rng, start=(0, 0, 0))
        if c[0, 0] > c[1:, 0].max() + 0.02:
            break
    c += lo + np.array([2*L + 0.01 - c[0, 0], 0.5*L, 0.5*L])
    assert c[0, 0] - lo[0] > 2*L > (c[1:, 0] - lo[0]).max()
    n = w.natoms
    d = systems.SystemDesc(**{k: v for k, v in w.__dict__.items()})
    d.masses = np.concatenate([w.masses, np.full(5, 12.0)])
    d.charges = np.concatenate([w.charges, np.zeros(5)])
    d.sigmas = np.concatenate([w.sigmas, np.full(5, 0.3)])
    d.epsilons = np.concatenate([w.epsilons, np.zeros(5)])
    d.positions = np.concatenate([w.positions, c]).astype(np.float32).astype(np.float64)
    size, energy, coeff = _maps()
    d.cmap_atoms = np.array([[n, n+1, n+2, n+3, n+1, n+2, n+3, n+4]], dtype=np.int32)
    d.cmap_size, d.cmap_energy, d.cmap_coeff, d.cmap_map = size[:1], energy[:576], coeff[:576], np.zeros(1, np.int32)
    pme = d.pme_parameters()
    eng = Engine(d)
    e = eng.compute()
    f = eng.get_forces()
    assert np.abs(eng.get_positions() - d.positions).max() < 1e-5          # the user still sees the positions set
    fr, er = harness.Simulation(d, "Reference", pme=pme).forces_energy()
    assert relative_force_error(f, fr) < 1e-4 and abs(e - er)/abs(er) < 1e-4
    assert np.abs(f[n:] - fr[n:]).max() <= 1e-6*max(1.0, np.abs(fr[n:]).max())


# ---------------------------------------------------------------------------------------------------- through the plugin
def test_plugin_runs_dhfr_cmap_rb(harness, dhfr):
    from openmm_b200 import systems
    pme = dhfr.pme_parameters()
    v = np.random.default_rng(3).standard_normal((dhfr.natoms, 3))*0.3
    runs = {}
    for platform, fused in (("Reference", None), ("B200", "1"), ("B200", "0")):
        if fused is not None:
            os.environ["B200MD_PLUGIN_FUSED"] = fused
        try:
            s = harness.Simulation(dhfr, platform, integrator=(systems.INT_VERLET, 0, 0, 0.001), pme=pme)
        finally:
            os.environ.pop("B200MD_PLUGIN_FUSED", None)
        assert s.platform() == platform
        s.set_velocities(v)
        s.step(20)
        runs[(platform, fused)] = s.state(positions=True)["positions"]
        s.close()
    # both step paths follow the Reference platform: a path that skipped the RB or CMAP forces would be ~1e-4 nm off by now.
    # The two paths are not bit-equal (test_gpu_plugin.py bounds them by 2e-6 nm on water).
    for fused in ("1", "0"):
        assert np.abs(runs[("B200", fused)] - runs[("Reference", None)]).max() < 5e-6, fused
    assert np.abs(runs[("B200", "1")] - runs[("B200", "0")]).max() < 5e-6
    s = harness.Simulation(dhfr, "B200", integrator=(systems.INT_LANGEVIN_MIDDLE, 300.0, 1.0, 0.002), pme=pme)
    s.set_velocities_to_temperature(300.0, 4)
    s.step(1000)
    x = s.state(positions=True)["positions"]
    assert np.isfinite(x).all()
    for i, j, dist in zip(dhfr.con_i[::7], dhfr.con_j[::7], dhfr.con_d[::7]):
        assert abs(np.linalg.norm(x[i]-x[j]) - dist) < 1e-4*dist


# ---------------------------------------------------------------------------------------------------- multi-GPU
_WORKER = r"""
import os, sys, ctypes as C
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, os.path.join(sys.argv[1], "tests"))
import numpy as np, torch, torch.distributed as dist
from openmm_b200 import Engine, _lib
from test_gpu_cmap_rb import dhfr_cmap_rb
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("gloo")
os.environ.setdefault("B200MD_NCCL_LIB", os.path.join(os.path.dirname(torch.__file__), "..", "nvidia", "nccl", "lib", "libnccl.so.2"))
uid = torch.zeros(128, dtype=torch.uint8)
if rank == 0:
    buf = C.create_string_buffer(128)
    assert _lib.load().b200md_comm_unique_id(C.cast(buf, C.c_void_p)) == 0
    uid = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
dist.broadcast(uid, 0)
d = dhfr_cmap_rb()
ref = Engine(d, device=local); ref.compute(); fref = ref.get_forces()
eng = Engine(d, device=local, comm=(rank, world, bytes(uid.numpy().tobytes()))); eng.compute(); f = eng.get_forces()
if rank == 0:
    print("CMAP_RB_MULTI max|dF| = %g" % float(np.abs(f - fref).max()))
dist.barrier()
"""


def test_multi_gpu_forces_equal_single_gpu(tmp_path):
    import torch
    n = torch.cuda.device_count() if torch.cuda.is_available() else 0
    if n < 2:
        pytest.skip("needs 2 GPUs on one machine, this one has %d" % n)
    worker = tmp_path / "cmap_rb_worker.py"
    worker.write_text(_WORKER)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc-per-node", "2", "--master-port", "29432", str(worker), ROOT]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "CMAP_RB_MULTI max|dF| = 0\n" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
