"""GPU tests of the potential energy and of energy differences at the kT scale, against the double-precision restatement
(tests/energy_harness.py) given exactly the fp32 coordinates the kernels read:
 A. each term mask's energy on the proteins, the water and ion boxes, the edge systems of tests/test_gpu_oracle_edges.py,
    the non-PME methods and LJ-only / Coulomb-only water;
 B. the energy change of barostat moves of 1e-4 to 1e-2 in volume, through host-built positions and through the engine's
    own scale_coordinates + set_box;
 C. the energy change of NonbondedForce parameter changes along lambda;
 D. energies of frames of a run on an aged neighbour list;
 E. the same through the OpenMM plugin, against the Reference platform in the same process.
Where the energy matters most it is a small difference of large numbers (the barostat's w = dE + P dV - N kT ln(V'/V),
E/kT at every lambda of a free-energy run): energy differences are held to 0.1 kT, totals to 1 kT."""
import copy
import os
import numpy as np
import pytest
from conftest import ROOT
import energy_harness as EH
import test_gpu_oracle_edges as edges

pytestmark = pytest.mark.gpu
PRECISIONS = ["single", "mixed"]
KT = EH.KT
DE_BOUND = 0.1*KT                # an energy difference: barostat acceptance, lambda windows
TOTAL_BOUND = 1.0*KT             # a total energy
BONDED_REL = 1e-9                # bonded parts: double on both sides, relative to max(1, |part|)
# Absolute bounds in kJ/mol on the direct (TERM_NB_DIRECT) and reciprocal (TERM_NB_RECIP) parts against the oracle, per
# system: twice the worst error measured over both precisions and four runs on an H100 SXM (80 GB HBM3, 700 W power
# limit), and no less than PART_FLOOR.  The measured worst errors (direct, reciprocal; "-": no PME):
#   dhfr 0.1227, 0.0003         apoa1 0.2248, 0.0009 (0.219-0.225 from run to run: the order in which the tile kernel's
#   warps add their fp32 totals varies)    water24k 0.7595, <1e-4    ions_triclinic 0.0071, 0.0221
#   shift_off 0.0213, <1e-4     shift_on 0.3678, <1e-4     pme_switch_water 0.0482, <1e-4     lj_short_switch 1e-4, -
#   close_contact_ions 0.0008, 0.0032     triclinic_pmp 0.0043, 0.0044     triclinic_mpm 0.0010, 0.0067
#   overflow_cluster <1e-4, -   reaction_field 0.0021, -   nocutoff 0.0003, -   cutoff_nonperiodic 0.0001, -
#   water24k_lj_only 0.0013, <1e-4    water24k_coulomb_only 0.7615, <1e-4    water7_lj_only 0.0002, <1e-4
#   water7_coulomb_only 0.0316, <1e-4    dhfr_frames (part D, 20 frames of two runs) 0.1479, 0.0003
#   water_flexible (part E, the plugin against the Reference platform) 0.0315, <1e-4
# PART_FLOOR covers the 1e-4 resolution of those measurements and the run-to-run spread of the fp32 sums.
PART_FLOOR = 5e-3
MEASURED = {"dhfr": (0.1227, 0.0003), "apoa1": (0.2248, 0.0009), "water24k": (0.7595, 0.0), "ions_triclinic": (0.0071, 0.0221),
            "shift_off": (0.0213, 0.0), "shift_on": (0.3678, 0.0), "pme_switch_water": (0.0482, 0.0), "lj_short_switch": (0.0001, 0.0),
            "close_contact_ions": (0.0008, 0.0032), "triclinic_pmp": (0.0043, 0.0044), "triclinic_mpm": (0.0010, 0.0067),
            "overflow_cluster": (0.0, 0.0), "reaction_field": (0.0021, 0.0), "nocutoff": (0.0003, 0.0), "cutoff_nonperiodic": (0.0001, 0.0),
            "water24k_lj_only": (0.0013, 0.0), "water24k_coulomb_only": (0.7615, 0.0), "water7_lj_only": (0.0002, 0.0),
            "water7_coulomb_only": (0.0316, 0.0), "dhfr_frames": (0.1479, 0.0003), "water_flexible": (0.0315, 0.0)}


def part_bounds(name):
    """(direct, reciprocal) bound in kJ/mol of system `name`"""
    return tuple(max(2.0*m, PART_FLOOR) for m in MEASURED[name])


# An aged list against a freshly built one at the same posq.  Each engine's energy repeats to 7e-9 kJ/mol, but the two
# lists group the pairs into different tiles, so the tile kernel's fp32 sums round differently: over 120 DHFR frames (three
# runs of 20 frames per precision, measured on the same H100) the difference has an rms of 2.5e-3 kJ/mol (single; mixed
# 2.1e-3) and is at most 1.2e-2.  FRESH_SUM_BOUND is six times that rms.  A pair within an fp32 rounding of its displacement
# of the cutoff may also fall on different sides of it in the two lists (the single-image shift is added to whichever atom
# the tile holds).  That costs one more rounding of each component; in the 6.2 nm DHFR box a shifted coordinate of a pair
# inside the cutoff stays below 8 nm, so the rounding is at most 2.4e-7 nm per component and 4.2e-7 nm along the pair.
# Every pair within EDGE_DELTA of the cutoff adds its |energy| to the bound of its frame (EH.cutoff_edge_energy; 0.04 to
# 0.1 kJ/mol on DHFR).
FRESH_SUM_BOUND = 0.015
EDGE_DELTA = 5e-7
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")


def _engine(d, precision):
    from openmm_b200 import Engine
    return Engine(d, precision=precision)


# ---------------------------------------------------------------- A. energies part by part
_SYSTEMS = {}


def _reference_case(name):
    from openmm_b200 import systems
    from test_gpu_parity import reference_cases
    return reference_cases(systems)[name]


def _only(d, what):
    """a copy of d with its charges (what = "lj") or its epsilons (what = "coulomb") set to zero"""
    d = copy.copy(d)
    if what == "lj":
        d.charges = np.zeros(d.natoms)
    else:
        d.epsilons = np.zeros(d.natoms)
    d.name = d.name + "_" + what
    return d


BUILDERS = {
    "dhfr": lambda s: EH.load("dhfr"), "apoa1": lambda s: EH.load("apoa1"), "water24k": lambda s: EH.load("water24k"),
    "ions_triclinic": lambda s: EH.load("ions_triclinic"),
    "shift_off": lambda s: edges.shift_box_pair(s)[0], "shift_on": lambda s: edges.shift_box_pair(s)[1],
    "pme_switch_water": edges.pme_switch_water, "lj_short_switch": edges.lj_short_switch,
    "close_contact_ions": edges.close_contact_ions, "triclinic_pmp": lambda s: edges.triclinic_limit_ions(s, "pmp"),
    "triclinic_mpm": lambda s: edges.triclinic_limit_ions(s, "mpm"), "overflow_cluster": edges.overflow_cluster,
    "reaction_field": lambda s: _reference_case("reaction_field"), "nocutoff": lambda s: _reference_case("nocutoff_cluster"),
    "cutoff_nonperiodic": lambda s: _reference_case("cutoff_nonperiodic"),
    "water24k_lj_only": lambda s: _only(EH.load("water24k"), "lj"), "water24k_coulomb_only": lambda s: _only(EH.load("water24k"), "coulomb"),
    "water7_lj_only": lambda s: _only(EH.load("water_rigid"), "lj"), "water7_coulomb_only": lambda s: _only(EH.load("water_rigid"), "coulomb"),
}


def _system(name):
    from openmm_b200 import systems
    if name not in _SYSTEMS:
        _SYSTEMS[name] = BUILDERS[name](systems)
    return _SYSTEMS[name]


def _check_parts(label, bounds, e, r, total, rtotal):
    """assert part and total bounds (bounds: part_bounds of the system); print the errors"""
    errs = {g: e[g] - r[g] for g in e}
    print("%s: %s; total %+.4f kJ/mol (%+.3f kT)" % (label, ", ".join("%s %+.4f" % kv for kv in errs.items()), total - rtotal,
                                                     (total - rtotal)/KT))
    for g, err in errs.items():
        if g in ("bonds", "angles", "torsions"):
            assert abs(err) <= BONDED_REL*max(1.0, abs(r[g])), (g, err)
        elif g == "direct":
            assert abs(err) <= bounds[0], (g, err, bounds)
        else:
            assert abs(err) <= bounds[1], (g, err, bounds)
    assert abs(total - rtotal) <= TOTAL_BOUND, (total, rtotal)


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(BUILDERS))
def test_energy_parts_match_oracle(name, precision):
    d = _system(name)
    eng = _engine(d, precision)
    e = EH.engine_parts(eng, d)
    total = eng.compute()
    assert eng.stats()["overflow"] == 0
    r = EH.oracle_parts(d, EH.kernel_positions(eng))
    _check_parts("%s %s" % (name, precision), part_bounds(name), e, r, total, sum(r.values()))


# ---------------------------------------------------------------- B. barostat moves
BAROSTAT = {"dhfr": EH.RUNGS, "water24k": EH.RUNGS, "ions_triclinic": EH.RUNGS, "lj_switch_dispersion": EH.RUNGS,
            "apoa1": ("+0.01", "-0.01", "aniso")}


def _energies(eng, d):
    e = EH.engine_parts(eng, d)
    e["total"] = eng.compute()
    return e


def _check_move(label, e0, e1, r0, r1):
    """e0 / e1 carry the engine's total under "total" (one evaluation of every term); r0 / r1 the oracle groups"""
    errs = {g: (e1[g] - e0[g]) - (r1[g] - r0[g]) for g in r1 if g in e1}
    de_r = sum(r1.values()) - sum(r0.values())
    err = (e1["total"] - e0["total"]) - de_r
    print("%s: dE %+.3f kJ/mol, error %+.5f kJ/mol (%+.4f kT); parts %s" % (label, de_r, err, err/KT,
                                                                           ", ".join("%s %+.5f" % kv for kv in errs.items())))
    assert abs(err) <= DE_BOUND, (label, err)
    return err


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", list(BAROSTAT))
def test_barostat_moves_host_positions(name, precision):
    """Each rung's configuration built on the host (fp32 positions and box) and given through set_positions + set_box."""
    d = EH.pinned_pme(EH.load(name))
    eng = _engine(d, precision)
    e0 = _energies(eng, d)
    r0 = EH.oracle_parts(d, EH.kernel_positions(eng))
    for rung in BAROSTAT[name]:
        dn, _ = EH.scaled(d, rung)
        eng.set_positions(dn.positions)
        eng.set_box(dn.box)
        e1 = _energies(eng, dn)
        r1 = EH.oracle_parts(dn, EH.kernel_positions(eng))
        _check_move("%s %s host %s" % (name, precision, rung), e0, e1, r0, r1)
    assert eng.stats()["overflow"] == 0


# ApoA1 goes through the engine's own scaling in single precision only: the posq that path produces is new to the oracle,
# and each ApoA1 oracle evaluation takes most of a minute (its host-built moves run in both precisions).
ENGINE_SCALING = [(n, p) for n in BAROSTAT for p in PRECISIONS if (n, p) != ("apoa1", "mixed")]


@pytest.mark.parametrize("name,precision", ENGINE_SCALING)
def test_barostat_moves_engine_scaling(name, precision):
    """Each rung through the engine's own scale_coordinates + set_box(scaled box) and, after it, restore_coordinates +
    set_box(box), as MonteCarloBarostatImpl moves and rejects; the oracle sees the posq the move produced.  After the last
    rejected move the energy is the first one again, up to the order of the tile kernel's fp32 sums."""
    d = EH.pinned_pme(EH.load(name))
    eng = _engine(d, precision)
    eng.set_barostat_molecules()
    e0 = _energies(eng, d)
    r0 = EH.oracle_parts(d, EH.kernel_positions(eng))
    for rung in BAROSTAT[name]:
        s = EH.rung_scale(rung)
        dn = copy.copy(d)
        dn.box = EH.scale_box(d.box, s)
        eng.scale_coordinates(*s)
        eng.set_box(dn.box)
        e1 = _energies(eng, dn)
        r1 = EH.oracle_parts(dn, EH.kernel_positions(eng))
        _check_move("%s %s engine %s" % (name, precision, rung), e0, e1, r0, r1)
        eng.restore_coordinates()
        eng.set_box(d.box)
    # the positions are restored bit for bit and the list is rebuilt from them: only the fp32 sums may round differently
    assert abs(eng.compute() - e0["total"]) <= FRESH_SUM_BOUND
    assert eng.stats()["overflow"] == 0


# ---------------------------------------------------------------- C. parameter changes
@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("system_name", ["dhfr", "ions_triclinic"])
def test_lambda_ladder(system_name, precision):
    """Every change of tests/nonbonded_params_harness.py at lambda = 0.25 ... 1 through update_nonbonded_params, dE from
    lambda = 0 (the dispersion coefficient stays that of lambda = 0)."""
    for change in EH.lambda_changes(system_name):
        d0, disp = EH.at_lambda(system_name, change, 0.0)
        eng = _engine(d0, precision)
        e0 = _energies(eng, d0)
        x = EH.kernel_positions(eng)
        r0 = EH.oracle_parts(d0, x, disp)
        for lam in EH.LAMBDAS[1:]:
            dl, _ = EH.at_lambda(system_name, change, lam)
            eng.update_nonbonded_params(dl, disp)
            e1 = _energies(eng, dl)
            _check_move("%s %s %s lambda %.2f" % (system_name, precision, change, lam), e0, e1, r0, EH.oracle_parts(dl, x, disp))
        assert eng.stats()["overflow"] == 0


# ---------------------------------------------------------------- D. aged lists
@pytest.mark.parametrize("precision", PRECISIONS)
def test_aged_list_frames(precision):
    """200 LangevinMiddle steps of DHFR, a frame every 20: each frame's parts against the oracle at its posq, its total against
    a freshly built engine at the same posq, and each frame-to-frame dE against the oracle's."""
    from openmm_b200 import systems
    d = EH.load("dhfr")
    eng = _engine(d, precision)
    eng.set_integrator(systems.INT_LANGEVIN_MIDDLE, 0.002, 300.0, 1.0, 11)
    eng.set_velocities(edges._thermal_velocities(d, 300.0, 11))
    eng.apply_velocity_constraints()
    prev = None
    worst_fresh = worst_margin = 0.0
    builds0 = eng.stats()["list_builds"]
    for k in range(10):
        eng.step(20)
        e = _energies(eng, d)
        x = EH.kernel_positions(eng)
        r = EH.oracle_parts(d, x)
        _check_parts("dhfr %s frame %d" % (precision, k), part_bounds("dhfr_frames"), {g: e[g] for g in r if g in e}, r, e["total"],
                     sum(r.values()))
        fd = copy.copy(d)
        fd.positions = x
        fresh = _engine(fd, precision)
        e_fresh = fresh.compute()
        fresh.close()
        bound = FRESH_SUM_BOUND + EH.cutoff_edge_energy(d, x, EDGE_DELTA)
        worst_fresh = max(worst_fresh, abs(e["total"] - e_fresh))
        worst_margin = max(worst_margin, abs(e["total"] - e_fresh)/bound)
        assert abs(e["total"] - e_fresh) <= bound, (k, e["total"] - e_fresh, bound)
        if prev is not None:
            _check_move("dhfr %s frames %d-%d" % (precision, k - 1, k), prev[0], e, prev[1], r)
        prev = (e, r)
    print("dhfr %s: %d list builds; aged list against a fresh one: at most %.2e kJ/mol, %.2f of its bound"
          % (precision, eng.stats()["list_builds"] - builds0, worst_fresh, worst_margin))
    assert eng.stats()["overflow"] == 0


# ---------------------------------------------------------------- E. through the plugin
@pytest.fixture(scope="module")
def omm():
    from oracle import omm
    if not omm.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where /root/reference exists")
    omm.load_plugin(PLUGIN)
    return omm


GROUPS = {"direct": 1, "reciprocal": 2, "bonded": 4}       # NonbondedForce in group 0, its reciprocal space in 1, bonded in 2


def _pair(omm, d, precision, **kw):
    from openmm_b200 import systems
    pme = d.pme_parameters() if d.method == systems.NB_PME else None
    return (omm.Simulation(d, "B200", props="Precision=" + precision, pme=pme, recip_group=1, bonded_group=2, **kw),
            omm.Simulation(d, "Reference", pme=pme, recip_group=1, bonded_group=2, **kw))


def _group_energies(sim):
    out = {g: sim.forces_energy(mask)[1] for g, mask in GROUPS.items()}
    out["total"] = sim.forces_energy()[1]
    return out


PLUGIN_SYSTEMS = ["water_flexible", "ions_triclinic", "dhfr"]


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("name", PLUGIN_SYSTEMS)
def test_plugin_group_energies_and_barostat_moves(omm, name, precision):
    """Per-force-group energies against the Reference platform's, then dE across Context::setPeriodicBoxVectors +
    setPositions (the calls MonteCarloBarostatImpl makes) on the 1e-2 and 1e-3 rungs (DHFR: one rung; the triclinic ion
    box: the growing ones, where the Reference platform's neighbour list is complete, EH.REFERENCE_LIST_MISSES)."""
    d = EH.pinned_pme(EH.load(name))
    a, b = _pair(omm, d, precision)
    ea, eb = _group_energies(a), _group_energies(b)
    errs = {g: ea[g] - eb[g] for g in ea}
    print("plugin %s %s: %s" % (name, precision, ", ".join("%s %+.4f" % kv for kv in errs.items())))
    direct_bound, recip_bound = part_bounds(name)
    assert abs(errs["direct"]) <= direct_bound and abs(errs["reciprocal"]) <= recip_bound
    assert abs(errs["bonded"]) <= BONDED_REL*max(1.0, abs(eb["bonded"])) + 1e-9
    assert abs(errs["total"]) <= TOTAL_BOUND
    rungs = ("-0.01",) if name == "dhfr" else ("+0.01", "-0.01", "+0.001", "-0.001")
    for rung in [r for r in rungs if (name, r) not in EH.REFERENCE_LIST_MISSES]:
        dn, _ = EH.scaled(d, rung)
        for s in (a, b):
            s.set_box(dn.box)
            s.set_positions(dn.positions)
        ea1, eb1 = _group_energies(a), _group_energies(b)
        err = (ea1["total"] - ea["total"]) - (eb1["total"] - eb["total"])
        print("plugin %s %s %s: dE %+.3f kJ/mol, error %+.5f kJ/mol (%+.4f kT)" % (name, precision, rung, eb1["total"] - eb["total"],
                                                                                err, err/KT))
        assert abs(err) <= DE_BOUND
        for s in (a, b):
            s.set_box(d.box)
            s.set_positions(d.positions)
    a.close()
    b.close()


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("system_name", ["water_rigid", "ions_triclinic"])
def test_plugin_set_parameter_lambda_ladder(omm, system_name, precision):
    """Context::setParameter of the parameter offsets of every change at once, along the lambda ladder: dE from lambda = 0."""
    import nonbonded_params_harness as NP
    base, p_off, e_off = NP.change(NP.system(system_name), "all")
    a, b = _pair(omm, base, precision, nb_globals={NP.LAM: 0.0}, particle_offsets=p_off, exception_offsets=e_off)
    e0 = [s.forces_energy()[1] for s in (a, b)]
    for lam in EH.LAMBDAS[1:]:
        for s in (a, b):
            s.set_parameter(NP.LAM, lam)
        e1 = [s.forces_energy()[1] for s in (a, b)]
        err = (e1[0] - e0[0]) - (e1[1] - e0[1])
        print("plugin %s %s lambda %.2f: dE %+.3f kJ/mol, error %+.5f kJ/mol (%+.4f kT)" % (system_name, precision, lam, e1[1] - e0[1],
                                                                                         err, err/KT))
        assert abs(err) <= DE_BOUND
    a.close()
    b.close()
