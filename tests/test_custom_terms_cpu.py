"""CPU tests of the custom-bond and custom-external expression programs: the plugin's translator (plugin/custom_translate.h) and
the interpreter the device kernel runs (openmm_b200/csrc/custom_interp.h), reached without a device through
b200md_custom_term_probe, against Lepton's own evaluation of the same expressions (periodicdistance: the Reference platform's
ReferencePointDistanceFunction); and the checks a program set of each class gets."""
import numpy as np
import pytest

OP_THETA, OP_PARAM, OP_VAR, OP_PERIODIC_DIST = 1, 2, 42, 43
BOX_ORTHO = np.diag([3.1, 2.7, 3.5])
BOX_TRICLINIC = np.array([[3.0, 0.0, 0.0], [0.9, 2.8, 0.0], [-0.7, 1.1, 3.3]])


@pytest.fixture(scope="module")
def harness():
    import custom_harness
    if not custom_harness.available():
        pytest.fail("oracle/_ref is not built: run __graft_entry__.build() where /root/reference exists")
    return custom_harness


def _run(h, cls, expr, which, variables, box=np.eye(3), params=(), pv=(), globals_=(), gv=()):
    op, arg, imm, starts = h.translate(cls, expr, params, globals_)
    value, err = h.term_probe(cls, starts, op, arg, imm, len(params), len(globals_), which, variables, box, pv, gv)
    assert err is None, err
    return value


def _close(x, y, rel=1e-12):
    return x == y or abs(x - y) <= rel*max(abs(x), abs(y))


BOND_EXPRESSIONS = ["0.5*k*(r-r0)^2", "step(r-r0)*k*(r-r0)^2", "k*(1-exp(-a*(r-r0)))^2", "g*k/r^6 - sqrt(r)*log(r+a)"]


@pytest.mark.parametrize("expr", BOND_EXPRESSIONS)
def test_bond_programs_match_lepton(harness, expr):
    h = harness
    params, globals_ = ("k", "r0", "a"), ("g",)
    op, _, _, starts = h.translate(h.BOND, expr, params, globals_)
    assert len(starts) == 3 and OP_VAR in op.tolist() and OP_THETA not in op.tolist()
    rng = np.random.default_rng(len(expr))
    for _ in range(30):
        r, pv, gv = rng.uniform(0.05, 0.4), [rng.uniform(100, 900), rng.uniform(0.08, 0.3), rng.uniform(0.5, 3)], [rng.uniform(-2, 2)]
        for which in (0, 1):
            ours = _run(h, h.BOND, expr, which, [r], params=params, pv=pv, globals_=globals_, gv=gv)
            ref = h.lepton(h.BOND, expr, which, [r], params=params, pvals=pv, globals_=globals_, gvals=gv)
            assert _close(ours, ref), (expr, which, r, ours, ref)


EXTERNAL_EXPRESSIONS = ["k*periodicdistance(x, y, z, x0, y0, z0)^2", "k*((x-x0)^2+(y-y0)^2+(z-z0)^2)",
                        "k*periodicdistance(x0, y0, z0, x, y, z)", "g*periodicdistance(x, y0, 0.3*z, x0, y, z0)^3 + k*atan2(x, y)"]


@pytest.mark.parametrize("box", [BOX_ORTHO, BOX_TRICLINIC], ids=["orthorhombic", "triclinic"])
@pytest.mark.parametrize("expr", EXTERNAL_EXPRESSIONS)
def test_external_programs_match_lepton(harness, expr, box):
    """every derivative of periodicdistance, with the point asymmetric in all six arguments and images in every direction, so
    that a swapped argument order or a wrong reduction fails"""
    h = harness
    params, globals_ = ("k", "x0", "y0", "z0"), ("g",)
    op, arg, _, starts = h.translate(h.EXTERNAL, expr, params, globals_)
    assert len(starts) == 5
    if "periodicdistance" in expr:
        assert OP_PERIODIC_DIST in op.tolist()
    rng = np.random.default_rng(len(expr))
    for _ in range(25):
        x = rng.uniform(-8, 8, 3)
        pv = [rng.uniform(10, 900)] + rng.uniform(-4, 4, 3).tolist()
        gv = [rng.uniform(-2, 2)]
        for which in range(4):
            ours = _run(h, h.EXTERNAL, expr, which, x, box, params, pv, globals_, gv)
            ref = h.lepton(h.EXTERNAL, expr, which, x, box, params, pv, globals_, gv)
            assert _close(ours, ref), (expr, which, x, ours, ref)


def test_periodic_distance_opcode_derivatives(harness):
    """PERIODIC_DIST with every operand (-1..5) alone, against the Reference platform's function through Lepton"""
    h = harness
    expr = "periodicdistance(x, y, z, x0, y0, z0)"
    start = [0, 7, 8, 9, 10]
    for k in range(-1, 6):
        op = [OP_PARAM, OP_PARAM, OP_PARAM, OP_VAR, OP_VAR, OP_VAR, OP_PERIODIC_DIST, OP_VAR, OP_VAR, OP_VAR]
        arg = [2, 1, 0, 2, 1, 0, k, 0, 1, 2]
        x, p = np.array([2.9, -3.3, 7.1]), np.array([0.2, 1.4, -0.6])
        for box in (BOX_ORTHO, BOX_TRICLINIC):
            value, err = h.term_probe(h.EXTERNAL, start, op, arg, [0.0]*10, 3, 0, 0, x, box, p, [])
            assert err is None, err
            if k < 3:
                ref = h.lepton(h.EXTERNAL, expr, k + 1, x, box, ("x0", "y0", "z0"), p)
            else:                       # d/dx0 = -d/dx
                ref = -h.lepton(h.EXTERNAL, expr, k - 2, x, box, ("x0", "y0", "z0"), p)
            assert _close(value, ref), (k, value, ref)


def test_periodic_distance_derivatives_are_zero_at_zero_distance(harness):
    h = harness
    expr = "k*periodicdistance(x, y, z, x0, y0, z0)"
    params = ("k", "x0", "y0", "z0")
    for box in (BOX_ORTHO, BOX_TRICLINIC):
        x = np.array([0.4, -1.2, 2.2])
        pv = [5.0, 0.4, -1.2, 2.2]
        for which in range(4):
            assert _run(h, h.EXTERNAL, expr, which, x, box, params, pv) == 0.0, which
        # a lattice vector away: the reduction leaves rounding residues, and the values are then the Reference platform's
        for shift in (box[0] - box[2], 2*box[1]):
            for which in range(4):
                v = _run(h, h.EXTERNAL, expr, which, x + shift, box, params, pv)
                assert not np.isnan(v) and _close(v, h.lepton(h.EXTERNAL, expr, which, x + shift, box, params, pv)), (which, v)


def test_limits_and_functions_are_refusals(harness):
    h = harness
    with pytest.raises(h.Refused):
        h.translate(h.BOND, "r", tuple("p%d" % k for k in range(17)))
    with pytest.raises(h.Refused):
        h.translate(h.EXTERNAL, "+".join("sin(%d*x)" % k for k in range(1, 120)))
    with pytest.raises(ValueError, match="Unknown variable"):
        h.translate(h.BOND, "r + theta")
    with pytest.raises(ValueError, match="Unknown variable"):
        h.translate(h.EXTERNAL, "x + r")


# ---------------------------------------------------------------------------------------------------- malformed programs
@pytest.mark.parametrize("cls,op,arg,match", [
    (1, [OP_VAR], [1], "custom bond program: variable index out of range for the class"),
    (1, [OP_VAR], [-1], "custom bond program: variable index out of range for the class"),
    (2, [OP_VAR], [3], "custom external program: variable index out of range for the class"),
    (1, [OP_THETA], [0], "custom bond program: THETA outside a torsion program"),
    (2, [OP_THETA], [0], "custom external program: THETA outside a torsion program"),
    (0, [OP_VAR], [0], "custom torsion program: unknown opcode"),
    (1, [OP_VAR]*6 + [OP_PERIODIC_DIST], [0]*6 + [-1], "PERIODIC_DIST outside an external program"),
    (2, [OP_VAR]*6 + [OP_PERIODIC_DIST], [0]*6 + [6], "periodic distance operand outside -1..5"),
    (2, [OP_VAR]*6 + [OP_PERIODIC_DIST], [0]*6 + [-2], "periodic distance operand outside -1..5"),
    (2, [OP_VAR]*5 + [OP_PERIODIC_DIST], [0]*5 + [0], "stack underflow"),
])
def test_malformed_programs_are_refused(harness, cls, op, arg, match):
    nv = harness.NUM_VARS[cls]
    # the malformed program first, then one VAR 0 (THETA for a torsion) per derivative
    good = OP_THETA if cls == 0 else OP_VAR
    ops, args = op + [good]*nv, arg + [0]*nv
    start = [0, len(op)] + [len(op) + k + 1 for k in range(nv)]
    value, err = harness.term_probe(cls, start, ops, args, [0.0]*len(ops), 0, 0, 0, [0.1, 0.2, 0.3], np.eye(3), [], [])
    assert value is None and match in err, err
