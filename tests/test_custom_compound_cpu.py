"""CPU tests of the custom-angle and custom-compound-bond expression programs: the plugin's translator (custom_translate.h)
and the interpreter (custom_interp.h, through b200md_custom_term_probe / b200md_custom_compound_probe) against Lepton
evaluating the prepared expression with the Reference platform's own point functions; degenerate geometry; malformed programs;
the limits validateSystem refuses."""
import math
import numpy as np
import pytest
import custom_harness as H

pytestmark = pytest.mark.skipif(not H.available(), reason="oracle/_ref (the built reference and the test C APIs) is absent")

ORTHO = np.diag([2.0, 2.5, 3.0])
TRICLINIC = np.array([[2.0, 0.0, 0.0], [0.4, 2.5, 0.0], [-0.3, 0.6, 3.0]])
POINT = {"pointdistance": 2, "pointangle": 3, "pointdihedral": 4}
OP = {"CONST": 0, "THETA": 1, "PARAM": 2, "ADD": 4, "MUL": 6, "VAR": 42, "PERIODIC_DIST": 43, "POINT_DIST": 44, "POINT_ANGLE": 45,
      "POINT_DIHEDRAL": 46}


def _close(a, b, tol=1e-12):
    return abs(a - b) <= tol*max(1.0, abs(b)) or (math.isnan(a) and math.isnan(b))


def _probe(nparticles, periodic, *rest):
    """b200md_custom_compound_probe (nparticles > 0) or b200md_custom_term_probe of the angle class"""
    return H.compound_probe(nparticles, periodic, *rest) if nparticles > 0 else H.term_probe(H.ANGLE, *rest)


def _check(nparticles, energy, x, box=np.eye(3), periodic=False, params=(), pvals=(), globals_=(), gvals=()):
    """every program of the expression through the probe against Lepton"""
    cls = H.COMPOUND if nparticles else H.ANGLE
    op, arg, imm, start = H.translate(cls, energy, params, globals_, nparticles)
    nprog = 1 + 3*nparticles if nparticles else 2
    assert len(start) == nprog + 1
    for which in range(nprog):
        got, msg = _probe(nparticles, periodic, start, op, arg, imm, len(params), len(globals_), which, x, box, pvals, gvals)
        assert msg is None, msg
        want = H.lepton(cls, energy, which, x, box, params, pvals, globals_, gvals, nparticles, periodic)
        assert _close(got, want), (energy, which, got, want)
    return op, arg, imm, start


@pytest.mark.parametrize("fn", sorted(POINT))
@pytest.mark.parametrize("box,periodic", [(ORTHO, False), (ORTHO, True), (TRICLINIC, True)], ids=["plain", "orthorhombic", "triclinic"])
def test_point_functions_match_reference_point_functions(fn, box, periodic):
    """value and every first derivative, the points spread over several cells so that differences straddle the box edges"""
    n = POINT[fn]
    args = ",".join("%s%d" % (a, i) for i in range(1, n + 1) for a in "xyz")
    rng = np.random.default_rng(5)
    for trial in range(6):
        x = rng.uniform(-1.0, 4.0, 3*n)
        _check(n, "%s(%s)" % (fn, args), x, box, periodic)


@pytest.mark.parametrize("periodic", [False, True])
def test_degenerate_geometry_returns_what_the_reference_returns(periodic):
    a = [0.3, 0.4, 0.5]
    # coincident points: distance 0 and zero derivatives
    _check(2, "distance(p1,p2)", a + a, ORTHO, periodic)
    # collinear angle, theta = pi and theta = 0
    _check(3, "angle(p1,p2,p3)", [0, 0, 0, 0.5, 0, 0, 1.0, 0, 0], ORTHO, periodic)
    _check(3, "angle(p1,p2,p3)", [0, 0, 0, 0.5, 0, 0, 0.2, 0, 0], ORTHO, periodic)
    # an angle with a zero-length arm: pi/2 by the reference's normed dot product
    _check(3, "angle(p1,p2,p3)", a + a + [0.9, 0.1, 0.2], ORTHO, periodic)
    # cis and trans dihedrals (0 and pi)
    _check(4, "dihedral(p1,p2,p3,p4)", [0, 0.5, 0, 0, 0, 0, 0.5, 0, 0, 0.5, 0.5, 0], ORTHO, periodic)
    _check(4, "dihedral(p1,p2,p3,p4)", [0, 0.5, 0, 0, 0, 0, 0.5, 0, 0, 0.5, -0.5, 0], ORTHO, periodic)


def test_dihedral_sign_convention():
    x = [0, 0.5, 0, 0, 0, 0, 0.5, 0, 0, 0.5, 0.3, 0.4]
    op, arg, imm, start = _check(4, "dihedral(p1,p2,p3,p4)", x)
    mirrored = list(x)
    mirrored[11] = -0.4
    v, _ = H.compound_probe(4, False, start, op, arg, imm, 0, 0, 0, x, np.eye(3), (), ())
    w, _ = H.compound_probe(4, False, start, op, arg, imm, 0, 0, 0, mirrored, np.eye(3), (), ())
    assert v == -w and v != 0.0


def test_realistic_expressions():
    from openmm_b200 import systems
    rng = np.random.default_rng(11)
    # the six-particle restraint
    _check(6, systems.ORIENTATIONAL_RESTRAINT, rng.uniform(0, 2, 18), ORTHO, False, systems.ORIENTATIONAL_PARAMS,
           [4000, 400, 400, 1.0, 1.5, 1.7, 0.3, -2.9, 3.0])
    _check(6, systems.ORIENTATIONAL_RESTRAINT, rng.uniform(-1, 4, 18), TRICLINIC, True, systems.ORIENTATIONAL_PARAMS,
           [4000, 400, 400, 1.0, 1.5, 1.7, 0.3, -2.9, 3.0])
    # the class header's example: an angle plus a distance
    _check(3, "0.5*(kangle*(angle(p1,p2,p3)-theta0)^2+kbond*(distance(p1,p3)-r0)^2)", rng.uniform(0, 1, 9), params=("kangle", "kbond", "theta0", "r0"),
           pvals=[1.0, 2.0, 2.1, 0.9])
    # the distance of a particle to the midpoint of two others
    _check(3, "k*pointdistance(x1, y1, z1, (x2+x3)/2, (y2+y3)/2, (z2+z3)/2)^2", rng.uniform(0, 1, 9), params=("k",), pvals=[3.0])
    # reads coordinates directly, globals and 16 per-bond parameters
    names = tuple("c%d" % i for i in range(16))
    _check(2, "lam*distance(p1,p2)*(" + "+".join(names) + ") + mu*x1 + 2*y2", rng.uniform(0, 1, 6), params=names, pvals=np.arange(16.0),
           globals_=("lam", "mu"), gvals=[0.3, 0.2])
    # the custom angle forms of coarse-grained force fields
    for theta in (0.0, 0.4, 2.0, math.pi):
        _check(0, "0.5*k*(cos(theta)-cos(theta0))^2", [theta], params=("k", "theta0"), pvals=[30.0, 1.9])
        _check(0, "0.5*k*(theta-theta0)^2 + lam*sin(theta)^2", [theta], params=("k", "theta0"), pvals=[30.0, 1.9], globals_=("lam",), gvals=[0.7])


def test_a_derivative_that_is_identically_zero_is_one_const():
    op, arg, imm, start = H.translate(H.COMPOUND, "distance(p1,p2)^2", nparticles=3)
    for q in range(7, 10):         # the programs of x3, y3, z3
        assert start[q+1] - start[q] == 1 and op[start[q]] == OP["CONST"] and imm[start[q]] == 0.0


def _one(nparticles, op, arg):
    """the programs `op` as the energy, CONST 0 for every derivative"""
    nder = 3*nparticles if nparticles else 1
    ops, args = list(op) + [OP["CONST"]]*nder, list(arg) + [0]*nder
    start = [0] + [len(op) + k for k in range(nder + 1)]
    return start, ops, args, [0.0]*len(ops)


@pytest.mark.parametrize("nparticles,op,arg,match", [
    (2, [OP["VAR"]], [6], "custom compound program: variable index out of range"),
    (2, [OP["VAR"]]*6 + [OP["POINT_DIST"]], [0, 1, 2, 3, 4, 5, 6], "custom compound program: point function operand out of range"),
    (4, [OP["VAR"]]*12 + [OP["POINT_DIHEDRAL"]], list(range(12)) + [-2], "custom compound program: point function operand out of range"),
    (2, [OP["VAR"]]*33 + [OP["ADD"]]*32, [0]*65, "custom compound program: stack deeper than 32"),
    (3, [OP["VAR"]]*8 + [OP["POINT_ANGLE"]], [0]*9, "custom compound program: stack underflow"),
    (2, [OP["THETA"]], [0], "custom compound program: THETA outside a torsion program"),
    (0, [OP["VAR"]], [0], "custom angle program: unknown opcode"),
    (0, [OP["THETA"]]*6 + [OP["PERIODIC_DIST"]], [0]*7, "custom angle program: unknown opcode"),
    (0, [OP["THETA"]]*17 + [OP["ADD"]]*16, [0]*33, "custom angle program: stack deeper than 16"),
])
def test_malformed_programs_are_refused(nparticles, op, arg, match):
    start, ops, args, imm = _one(nparticles, op, arg)
    got, msg = _probe(nparticles, False, start, ops, args, imm, 0, 0, 0, np.zeros(max(1, 3*nparticles)), np.eye(3), (), ())
    assert got is None and match in msg, msg


@pytest.mark.parametrize("cls,prefix", [(0, "custom torsion"), (1, "custom bond"), (2, "custom external")])
def test_point_opcodes_are_unknown_to_the_other_classes(cls, prefix):
    nvars = 3 if cls == 2 else 1
    var = OP["THETA"] if cls == 0 else OP["VAR"]
    ops = [var]*6 + [OP["POINT_DIST"]] + [OP["CONST"]]*nvars
    start = [0, 7] + [8 + k for k in range(nvars)]
    got, msg = H.term_probe(cls, start, ops, [0]*len(ops), [0.0]*len(ops), 0, 0, 0, np.zeros(3), np.eye(3), (), ())
    assert got is None and msg.startswith(prefix + " program: unknown opcode"), msg


def test_limits_are_refused_as_unsupported():
    nine = "+".join("x%d" % i for i in range(1, 10))
    with pytest.raises(H.Refused, match="more than 8 particles per bond"):
        H.translate(H.COMPOUND, nine, nparticles=9)
    names = tuple("c%d" % i for i in range(17))
    with pytest.raises(H.Refused, match="more than 16 per-bond parameters"):
        H.translate(H.COMPOUND, "distance(p1,p2)*(" + "+".join(names) + ")", names, nparticles=2)
    with pytest.raises(H.Refused, match="tabulated functions"):
        H.translate(H.COMPOUND, "fn(distance(p1,p2))", nparticles=2, tabulated=True)
    # 13 values under a dihedral call, each pair of parentheses one more: deeper than 32
    deep = "dihedral(p1,p2,p3,p4)"
    for k in range(24):
        deep = "x1*(y1+" + deep + ")"
    with pytest.raises(H.Refused, match="deeper than 32"):
        H.translate(H.COMPOUND, deep, nparticles=4)
    with pytest.raises(ValueError, match="Unknown variable"):
        H.translate(H.COMPOUND, "1+none", nparticles=2)
