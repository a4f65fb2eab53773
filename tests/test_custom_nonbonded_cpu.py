"""The CustomNonbondedForce class of the expression interpreter (custom_interp.h) on the host, through
b200md_custom_nonbonded_probe: the DISCRETE1/2/3 table lookups against ReferenceDiscrete{1,2,3}DFunction::evaluate restated in
numpy (round half away from zero, x + xsize (y + ysize z)), NaN for an index outside the table, a derivative of a table as 0,
the PARAM slots of the two particles, and the programs the class refuses."""
import ctypes as C

import numpy as np
import pytest

from openmm_b200 import _lib

OP = {"CONST": 0, "PARAM": 2, "GLOBAL": 3, "ADD": 4, "MUL": 6, "DIV": 7, "THETA": 1, "VAR": 42, "PERIODIC_DIST": 43,
      "DISCRETE1": 47, "DISCRETE2": 48, "DISCRETE3": 49}


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(C.POINTER(C.c_int))


def _d(a):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a, a.ctypes.data_as(C.POINTER(C.c_double))


def probe(programs, nparams, which, r, params, tables=(), globals_=(0.0,), nglobals=0):
    """programs: list of [(opcode name, operand, immediate)], two per object; tables: list of arrays of 1 to 3 dimensions
    (x = the first argument, fastest).  Returns (value, None) or (None, message)."""
    start = np.concatenate([[0], np.cumsum([len(p) for p in programs])])
    flat = [ins for p in programs for ins in p]
    op = [OP[o] for o, _, _ in flat]
    arg = [a for _, a, _ in flat]
    imm = [v for _, _, v in flat]
    dims, tstart, values = [], [0], []
    for t in tables:
        t = np.asarray(t, dtype=np.float64)
        shape = list(t.shape) + [1]*(3 - t.ndim)
        dims += [t.ndim] + shape
        values += list(t.transpose().ravel())          # x fastest
        tstart.append(len(values))
    keep = [_i(start), _i(op or [0]), _i(arg or [0]), _d(imm or [0.0]), _d(list(params) or [0.0]), _d(list(globals_)),
            _i(dims or [0]), _i(tstart), _d(values or [0.0])]
    out, msg = C.c_double(), C.create_string_buffer(256)
    rc = _lib.load().b200md_custom_nonbonded_probe(len(programs), keep[0][1], keep[1][1], keep[2][1], keep[3][1], nparams, nglobals, which,
                                                   r, keep[4][1], keep[5][1], len(tables), keep[6][1], keep[7][1], keep[8][1],
                                                   C.byref(out), msg, 256)
    return (out.value, None) if rc == 0 else (None, msg.value.decode())


def reference_lookup(table, args):
    """ReferenceDiscrete{1,2,3}DFunction::evaluate: C round() (halves away from zero); out of range raises there"""
    idx = tuple(int(np.sign(a)*np.floor(abs(a) + 0.5)) for a in args)
    if any(i < 0 or i >= n for i, n in zip(idx, table.shape)):
        return None
    return table[idx]


ZERO = [("CONST", 0, 0.0)]


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_discrete_tables_match_the_reference_lookup(ndim):
    rng = np.random.default_rng(ndim)
    shape = (5, 4, 3)[:ndim]
    table = rng.normal(size=shape)
    other = rng.normal(size=(2, 2))                   # table 0; the one looked up is table 1
    # arguments from the parameters: argument k is PARAM k, pushed last-first so that argument 0 is on top
    prog = [("PARAM", k, 0.0) for k in reversed(range(ndim))] + [("DISCRETE%d" % ndim, 1, 0.0)]
    for _ in range(200):
        args = rng.uniform(-0.7, np.array(shape) - 0.3)
        half = rng.random(ndim) < 0.3                 # exact halves: rounded away from zero
        args[half] = np.floor(args[half]) + 0.5
        params = list(args) + [0.0]*(2*ndim - ndim)
        v, err = probe([prog, ZERO], ndim, 0, 0.5, params, tables=[other, table])
        assert err is None, err
        want = reference_lookup(table, args)
        if want is None:
            assert np.isnan(v), (args, v)
        else:
            assert v == want, (args, v, want)


def test_rounding_and_out_of_range_give_nan_not_a_clamped_value():
    table = np.arange(4.0) + 10.0
    prog = [("PARAM", 0, 0.0), ("DISCRETE1", 0, 0.0)]
    for x, want in [(1.5, 12.0), (2.4999, 12.0), (-0.4, 10.0), (3.49, 13.0), (3.5, None), (-0.5, None), (1e9, None),
                    (float("nan"), None), (-7.0, None)]:
        v, err = probe([prog, ZERO], 1, 0, 0.5, [x, 0.0], tables=[table])
        assert err is None
        assert (np.isnan(v) if want is None else v == want), (x, v)


def test_derivative_of_a_table_is_zero():
    table = np.arange(9.0).reshape(3, 3)
    prog = [("PARAM", 1, 0.0), ("PARAM", 0, 0.0), ("DISCRETE2", -1, 0.0)]
    v, err = probe([ZERO, prog], 1, 1, 0.5, [1.0, 2.0], tables=[table])
    assert err is None and v == 0.0


def test_first_and_second_particle_parameter_slots():
    """PARAM k reads the first particle's parameter k, PARAM P+k the second's: p1*10 + p2 for every k of P = 3"""
    params = [1.0, 2.0, 3.0, 4.0, 5.0, 6.0]
    for k in range(3):
        prog = [("PARAM", k, 0.0), ("CONST", 0, 10.0), ("MUL", 0, 0.0), ("PARAM", 3 + k, 0.0), ("ADD", 0, 0.0)]
        # ADD/MUL take argument 0 = top of stack; the value does not depend on the order here
        v, err = probe([prog, ZERO], 3, 0, 0.5, params)
        assert err is None and v == params[k]*10 + params[3 + k]


def test_r_is_variable_zero():
    prog = [("VAR", 0, 0.0), ("VAR", 0, 0.0), ("MUL", 0, 0.0)]
    v, err = probe([prog, ZERO], 0, 0, 0.7, [])
    assert err is None and abs(v - 0.49) < 1e-15


@pytest.mark.parametrize("program, nparams, ntables, why", [
    ([("VAR", 1, 0.0)], 0, 0, "variable index out of range"),
    ([("THETA", 0, 0.0)], 0, 0, "THETA outside a torsion program"),
    ([("PARAM", 2, 0.0)], 1, 0, "parameter index out of range"),
    ([("PARAM", 0, 0.0), ("DISCRETE1", 1, 0.0)], 1, 1, "table index out of range"),
    ([("PARAM", 0, 0.0), ("DISCRETE1", -2, 0.0)], 1, 1, "table index out of range"),
    ([("PARAM", 0, 0.0), ("DISCRETE2", 0, 0.0)], 1, 1, "stack underflow"),
    ([("ADD", 0, 0.0)], 0, 0, "stack underflow"),
    ([("CONST", 0, 1.0), ("CONST", 0, 1.0)], 0, 0, "does not end with exactly one value"),
    ([("GLOBAL", 0, 0.0)], 0, 0, "global parameter index out of range"),
    ([("PARAM", 0, 0.0)], 9, 0, "more than 8 per-particle parameters"),
])
def test_malformed_programs_are_refused(program, nparams, ntables, why):
    tables = [np.zeros(2)]*ntables
    v, err = probe([program, ZERO], nparams, 0, 0.5, [0.0]*max(2*nparams, 1), tables=tables)
    assert v is None and why in err, err


def test_discrete_opcodes_belong_to_the_nonbonded_class_only():
    """a torsion or bond program with a DISCRETE instruction: an unknown opcode for those classes"""
    start, op, arg, imm = _i([0, 2, 3]), _i([OP["CONST"], OP["DISCRETE1"], OP["CONST"]]), _i([0, 0, 0]), _d([0.0, 0.0, 0.0])
    out, msg = C.c_double(), C.create_string_buffer(256)
    vars_, box, par, glob = _d([0.5]), _d(np.eye(3).ravel()), _d([0.0]), _d([0.0])
    for cls in (0, 1):
        rc = _lib.load().b200md_custom_term_probe(cls, 1, start[1], op[1], arg[1], imm[1], 0, 0, 0, vars_[1], box[1], par[1], glob[1],
                                                  C.byref(out), msg, 256)
        assert rc != 0 and "unknown opcode" in msg.value.decode()


# ---------------------------------------------------------------- the plugin's translator against Lepton, and the refusals
# Both need the reference's libOpenMM.so and the test C API (oracle/_ref), which __graft_entry__.build() makes where the
# reference sources exist.
import os  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PLUGIN = os.path.join(ROOT, "plugin", "libOpenMMB200.so")


@pytest.fixture(scope="module")
def H():
    import custom_nonbonded_harness
    if not custom_nonbonded_harness.available() or not os.path.exists(PLUGIN):
        pytest.fail("oracle/_ref or the plugin is not built: run __graft_entry__.build() where the reference sources exist")
    return custom_nonbonded_harness


# (expression, parameter names, tables {name: array}): the slots of p1 and p2 (asymmetric in the particles), every table
# dimension, a table's derivative (the tables' arguments are parameters: Lepton's chain rule multiplies it by 0), globals
EXPRESSIONS = [
    ("acoef(type1, type2)/r^12 - bcoef(type1, type2)/r^6", ["type"], {"acoef": (7, 7), "bcoef": (7, 7)}),
    ("a1*r + 2*b2 + a2^2*b1*exp(-r) + c1/r", ["a", "b", "c"], {}),
    ("t(k1)*r^2 + u(k1, k2, k1)*sqrt(r)", ["k"], {"t": (5,), "u": (5, 5, 5)}),
    ("s*w(k2, k1)*(r - r0)^2; r0 = 0.1*k1", ["k"], {"w": (4, 4)}),
    ("min(q1*q2/r, 10) + select(step(r - 0.5), 1, r)", ["q"], {}),
]


@pytest.mark.parametrize("case", range(len(EXPRESSIONS)))
def test_translated_programs_match_lepton(H, case):
    """translateNonbonded's energy and dE/dr programs, run by the interpreter, against Lepton evaluating the same expression
    with the Reference platform's Discrete*Function objects"""
    energy, names, shapes = EXPRESSIONS[case]
    rng = np.random.default_rng(case)
    n = 2
    f = H.Force(energy, names, np.zeros((n, len(names))), 0, 1.0, lrc=False, globals_={"s": 1.7} if "s*" in energy else None)
    s = H.Standalone(f, n)
    tables = {k: rng.normal(size=shape) for k, shape in shapes.items()}
    for k, t in tables.items():
        s.add_table(k, t)
    start, op, arg, imm, dims, tstart, values = s.translate()
    assert list(dims[:, 0]) == [len(tables[k].shape) for k in tables]
    inv = {v: k for k, v in OP.items()}
    for _ in range(50):
        P = len(names)
        maxk = min([min(t.shape) for t in tables.values()] + [4]) - 1
        p1, p2 = rng.integers(0, maxk + 1, P).astype(float), rng.integers(0, maxk + 1, P).astype(float)
        if not tables:
            p1, p2 = rng.uniform(0.2, 2.0, P), rng.uniform(0.2, 2.0, P)
        r = rng.uniform(0.3, 1.5)
        progs = [[(inv.get(o, o), a, v) for o, a, v in zip(op[start[q]:start[q+1]], arg[start[q]:start[q+1]], imm[start[q]:start[q+1]])]
                 for q in range(2)]
        for which in (0, 1):
            want = s.lepton(which, r, p1, p2)
            got, err = _probe_raw(start, op, arg, imm, P, which, r, list(p1) + list(p2), dims, tstart, values,
                                  [1.7] if "s*" in energy else [0.0], 1 if "s*" in energy else 0)
            assert err is None, err
            assert abs(got - want) <= 1e-12*max(1.0, abs(want)), (which, r, p1, p2, got, want, progs)
    s.close()


def _probe_raw(start, op, arg, imm, nparams, which, r, params, dims, tstart, values, globals_, nglobals):
    keep = [_i(start), _i(op), _i(arg), _d(imm), _d(params), _d(globals_), _i(np.asarray(dims).ravel() if len(dims) else [0]),
            _i(tstart), _d(values if len(values) else [0.0])]
    out, msg = C.c_double(), C.create_string_buffer(256)
    rc = _lib.load().b200md_custom_nonbonded_probe(len(start) - 1, keep[0][1], keep[1][1], keep[2][1], keep[3][1], nparams, nglobals, which,
                                                   r, keep[4][1], keep[5][1], len(dims), keep[6][1], keep[7][1], keep[8][1],
                                                   C.byref(out), msg, 256)
    return (out.value, None) if rc == 0 else (None, msg.value.decode())


def test_translator_refuses_continuous_tables_and_too_many_parameters(H):
    f = H.Force("r*k1", ["k"], np.zeros((2, 1)), 0, 1.0, lrc=False)
    s = H.Standalone(f, 2)
    assert H.lib().cnbc_add_continuous(s.sys, s.index, b"smooth") == 0
    with pytest.raises(RuntimeError, match="continuous tabulated functions"):
        s.translate()
    s.close()
    names = ["p%d" % k for k in range(9)]
    f = H.Force("r*(" + "+".join(p + "1*" + p + "2" for p in names) + ")", names, np.zeros((2, 9)), 0, 1.0, lrc=False)
    s = H.Standalone(f, 2)
    with pytest.raises(RuntimeError, match="more than 8 per-particle parameters"):
        s.translate()
    s.close()


# Every case validateSystem refuses, with its message, raised by contextCreated: the Context is created on the B200 platform by
# name, and the refusal comes before b200md_create (on a machine without a GPU, the matching System gets as far as that call).
REFUSALS = {
    "interaction_group": "interaction groups of a CustomNonbondedForce",
    "derivative": "energy parameter derivatives of a CustomNonbondedForce",
    "continuous": "continuous tabulated functions",
    "too_many_params": "more than 8 per-particle parameters",
    "two_cutoffs": "different methods or cutoffs",
    "two_methods": "different methods or cutoffs",
    "object_exclusions": "CustomNonbondedForce objects with different exclusions",
    "nb_exclusions": "exclusions differ from the NonbondedForce's exceptions",
    "nb_method": "nonbonded method does not match the NonbondedForce's",
    "nb_cutoff": "cutoff differs from the NonbondedForce's",
    "gbsa_beside_cutoff": "GBSAOBCForce beside a CustomNonbondedForce with a cutoff",
}


def refusal_case(H, case):
    """(desc, forces, after) of a refusal case on four particles: after(sim) adds what the C API adds to a built System"""
    from openmm_b200 import systems
    n = 4
    x = np.array([[0, 0, 0], [0.4, 0, 0], [0, 0.5, 0], [0, 0, 0.6]], dtype=np.float64)
    d = systems.SystemDesc(masses=np.full(n, 40.0), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n), positions=x,
                           method=systems.NB_NOCUTOFF, cutoff=1.0)
    f = H.Force("4*((0.3/r)^12-(0.3/r)^6)*a1*a2", ["a"], np.ones((n, 1)), 0, 1.0, lrc=False)
    forces, after = [f], []
    if case in ("two_cutoffs", "two_methods", "nb_cutoff"):
        d.method, f.method = systems.NB_CUTOFF_NONPERIODIC, 1
    if case == "two_cutoffs":
        forces.append(H.Force("r", [], np.zeros((n, 0)), 1, 0.9, lrc=False, group=3))
    if case == "two_methods":
        forces.append(H.Force("r", [], np.zeros((n, 0)), 0, 1.0, lrc=False, group=3))
    if case == "nb_cutoff":
        f.cutoff = 0.95
    if case == "object_exclusions":
        forces.append(H.Force("r", [], np.zeros((n, 0)), 0, 1.0, lrc=False, group=3, exclusions=[[0, 1]]))
    if case == "nb_exclusions":
        f.exclusions = np.array([[0, 1]], dtype=np.int32)
    if case == "nb_method":
        f.method = 1
    if case == "too_many_params":
        f.names = ["p%d" % k for k in range(9)]
        f.params = np.ones((n, 9))
        f.energy = "r*(" + "+".join("p%d1*p%d2" % (k, k) for k in range(9)) + ")"
    if case == "interaction_group":
        a, b = np.array([0, 1], dtype=np.int32), np.array([2, 3], dtype=np.int32)
        after.append(lambda sim: H.lib().cnbc_add_interaction_group(sim.sys, sim.cnb_index[0], 2, H._ip(a), 2, H._ip(b)))
    if case == "derivative":
        forces.append(H.Force("g*r", [], np.zeros((n, 0)), 0, 1.0, lrc=False, globals_={"g": 1.0}, group=3))
        after.append(lambda sim: H.lib().cnbc_add_derivative(sim.sys, sim.cnb_index[1], b"g"))
    if case == "continuous":
        after.append(lambda sim: H.lib().cnbc_add_continuous(sim.sys, sim.cnb_index[0], b"smooth"))
    if case == "gbsa_beside_cutoff":
        # no NonbondedForce's list to share: the custom force's (CutoffNonPeriodic) would cut the NoCutoff Born sums off
        d.method, f.method = systems.NB_NOCUTOFF, 1
        d.gb_charges, d.gb_radii, d.gb_scales = np.zeros(n), np.full(n, 0.15), np.full(n, 0.8)
    return d, forces, after


@pytest.mark.parametrize("case", sorted(REFUSALS))
def test_refusals_come_from_context_created_with_their_message(H, case):
    import gbsa_harness

    class Sim(H.Simulation):
        def add_forces(self):
            super().add_forces()
            for a in self.after:
                assert a(self) == 0

    d, forces, after = refusal_case(H, case)
    Sim.after = after
    H.omm.load_plugin(PLUGIN)
    if case == "gbsa_beside_cutoff":
        # a System without a NonbondedForce, built directly: a GBSAOBCForce at NoCutoff and the custom force
        L = H.omm.lib()
        sys_ = L.omm_system_create(d.natoms, H._dp(d.masses))
        assert gbsa_harness.lib().gbc_add_force(sys_, d.natoms, H._dp(d.gb_charges), H._dp(d.gb_radii), H._dp(d.gb_scales), 0, 1.0,
                                                1.0, 78.5, 2.25936, 4) >= 0
        forces[0].add_to(sys_)
        integ = L.omm_integrator_create(0, 0.0, 0.0, 0.001, 7, 1e-5)
        ctx = L.omm_context_create(sys_, integ, b"B200", b"")
        msg = L.omm_last_error().decode()
        if ctx:
            L.omm_context_destroy(ctx)
        L.omm_integrator_destroy(integ)
        L.omm_system_destroy(sys_)
        assert not ctx and "B200 platform: " in msg and REFUSALS[case] in msg, msg
        return
    with pytest.raises(RuntimeError) as e:
        Sim(d, "B200", forces=forces)
    assert "B200 platform: " in str(e.value) and REFUSALS[case] in str(e.value), str(e.value)
