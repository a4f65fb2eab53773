"""CPU tests of the custom-torsion expression programs: the plugin's translator (plugin/custom_translate.h) and the interpreter
the device kernel runs (openmm_b200/csrc/custom_interp.h), reached without a device through b200md_custom_program_probe,
against Lepton's own ExpressionProgram::evaluate of the same expressions; and the checks b200md_set_custom_torsions makes of
a program set, which the probe makes too."""
import math
import zlib
import numpy as np
import pytest
from openmm_b200 import systems
from custom_harness import program_probe as probe

OP = dict(CONST=0, THETA=1, PARAM=2, GLOBAL=3, ADD=4, SUB=5, MUL=6, DIV=7, POW=8, NEG=9, SQRT=10, EXP=11, LOG=12, SIN=13,
          COS=14, SEC=15, CSC=16, TAN=17, COT=18, ASIN=19, ACOS=20, ATAN=21, ATAN2=22, SINH=23, COSH=24, TANH=25, ERF=26,
          ERFC=27, STEP=28, DELTA=29, SQUARE=30, CUBE=31, RECIP=32, ADD_CONST=33, MUL_CONST=34, POW_CONST=35, MIN=36, MAX=37,
          ABS=38, FLOOR=39, CEIL=40, SELECT=41)
PARAMS, GLOBALS = ("a", "b"), ("g",)
# one expression per opcode, the arguments of the two-argument ones asymmetric, each followed by the opcode it must contain
EXPRESSIONS = [
    ("atan2(0.75, a*theta)", "CONST"), ("theta", "THETA"), ("a*theta", "PARAM"), ("g*theta", "GLOBAL"),
    ("a*theta + b*theta^2", "ADD"), ("a*sin(theta) - b*cos(theta)", "SUB"), ("sin(theta)*cos(a*theta)", "MUL"),
    ("sin(theta)/(b + cos(theta)^2)", "DIV"), ("(a + 0.1*theta)^(b*theta)", "POW"), ("-sin(theta)", "NEG"),
    ("sqrt(a + theta^2)", "SQRT"), ("exp(a*theta)", "EXP"), ("log(b + theta^2)", "LOG"), ("sin(a*theta)", "SIN"),
    ("cos(b*theta)", "COS"), ("sec(0.3*theta)", "SEC"), ("csc(0.2*theta + 1.5)", "CSC"), ("tan(0.4*theta)", "TAN"),
    ("cot(0.2*theta + 1.2)", "COT"), ("asin(0.3*theta)", "ASIN"), ("acos(0.3*theta)", "ACOS"), ("atan(a*theta)", "ATAN"),
    ("atan2(sin(theta), a + cos(theta))", "ATAN2"), ("sinh(0.5*theta)", "SINH"), ("cosh(0.5*theta)", "COSH"),
    ("tanh(a*theta)", "TANH"), ("erf(a*theta)", "ERF"), ("erfc(a*theta)", "ERFC"), ("step(theta - a)*theta^2", "STEP"),
    ("delta(floor(theta))*theta^2", "DELTA"), ("(theta - a)^2", "SQUARE"), ("(theta - b)^3", "CUBE"),
    ("1/(b + theta^2)", "RECIP"), ("theta + 2.5", "ADD_CONST"), ("3.5*theta", "MUL_CONST"), ("(b + theta^2)^1.7", "POW_CONST"),
    ("(1.3 + theta^2)^(-3)", "POW_CONST"), ("min(theta, a*cos(theta))", "MIN"), ("max(theta, a*cos(theta))", "MAX"),
    ("abs(theta - a)", "ABS"), ("floor(2*theta)*theta", "FLOOR"), ("ceil(2*theta)*theta", "CEIL"),
    ("select(step(theta), a*theta, b*theta^2)", "SELECT"),
]


@pytest.fixture(scope="module")
def harness():
    import custom_harness
    if not custom_harness.available():
        pytest.fail("oracle/_ref is not built: run __graft_entry__.build() where /root/reference exists")
    return custom_harness


def run(harness, expr, deriv, theta, pv, gv, params=PARAMS, globals_=GLOBALS):
    op, arg, imm, start = harness.translate(harness.TORSION, expr, params, globals_)
    value, err = probe(start, op, arg, imm, len(params), len(globals_), int(deriv), theta, pv, gv)
    assert err is None, err
    return value


def _close(x, y):
    return x == y or (np.isnan(x) and np.isnan(y)) or abs(x - y) <= 1e-14*max(abs(x), abs(y))


@pytest.mark.parametrize("expr,opname", EXPRESSIONS, ids=[e[0] for e in EXPRESSIONS])
def test_every_opcode_matches_lepton(harness, expr, opname):
    op, _, _, _ = harness.translate(harness.TORSION, expr, PARAMS, GLOBALS)
    assert OP[opname] in op.tolist(), (opname, op)
    rng = np.random.default_rng(zlib.crc32(expr.encode()))
    for _ in range(40):
        theta = rng.uniform(-math.pi, math.pi)
        pv, gv = rng.uniform(0.3, 1.8, 2), rng.uniform(-2.0, 2.0, 1)
        for deriv in (False, True):
            ours = run(harness, expr, deriv, theta, pv, gv)
            ref = harness.lepton(harness.TORSION, expr, deriv, [theta], params=PARAMS, pvals=pv, globals_=GLOBALS, gvals=gv)
            assert _close(ours, ref), (expr, deriv, theta, ours, ref)


def test_every_supported_opcode_is_covered():
    assert {name for _, name in EXPRESSIONS} == set(OP)


def test_derivative_program_is_leptons_derivative(harness):
    """the dE/dtheta program differs from the energy program and matches Lepton's derivative and a finite difference"""
    expr = "a*(1+cos(2*theta-b)) + g*sin(theta)^3"
    pv, gv = np.array([1.3, 0.4]), np.array([0.7])
    for theta in np.linspace(-3.1, 3.1, 23):
        de = run(harness, expr, True, theta, pv, gv)
        assert _close(de, harness.lepton(harness.TORSION, expr, True, [theta], params=PARAMS, pvals=pv, globals_=GLOBALS, gvals=gv))
        h = 1e-6
        fd = (run(harness, expr, False, theta + h, pv, gv) - run(harness, expr, False, theta - h, pv, gv))/(2*h)
        assert abs(fd - de) < 1e-7*max(1.0, abs(de))


def test_charmm_improper_across_the_seam(harness):
    """CharmmPsfFile's improper expression: near theta0 = +-pi the energy and its derivative follow the short way round"""
    expr, names = systems.CHARMM_IMPROPER, ("k", "theta0")
    pi6 = float("%f" % math.pi)
    for theta0 in (math.pi - 0.01, -math.pi + 0.02, 0.3):
        for theta in np.concatenate([np.linspace(-math.pi, -math.pi + 0.05, 6), np.linspace(math.pi - 0.05, math.pi, 6), [0.0, 1.0]]):
            pv = np.array([250.0, theta0])
            e, de = (run(harness, expr, d, theta, pv, [], names, ()) for d in (False, True))
            assert _close(e, harness.lepton(harness.TORSION, expr, False, [theta], params=names, pvals=pv))
            assert _close(de, harness.lepton(harness.TORSION, expr, True, [theta], params=names, pvals=pv))
            dt = abs(theta - theta0)
            short = min(dt, 2*pi6 - dt)
            assert abs(e - 250.0*short**2) <= 1e-12*max(1.0, e)
            sign = (1 if theta > theta0 else -1)*(1 if dt < 2*pi6 - dt else -1)
            assert abs(de - 2*250.0*short*sign) <= 1e-9*max(1.0, abs(de))


def test_unknown_variable_is_an_error_not_a_refusal(harness):
    with pytest.raises(ValueError, match="Unknown variable"):
        harness.translate(harness.TORSION, "theta+none", (), ())


def test_limits_are_refusals(harness):
    # Lepton pushes an operation's arguments last to first: nesting in the first argument deepens the stack one per level
    deep = "theta"
    for k in range(20):
        deep = "atan2(%s, theta)" % deep
    long_expr = "+".join("sin(%d*theta)" % k for k in range(1, 120))
    for expr, params in ((deep, ()), (long_expr, ()), ("theta", tuple("p%d" % k for k in range(17)))):
        try:
            op, _, _, _ = harness.translate(harness.TORSION, expr, params, ())
        except harness.Refused:
            continue
        pytest.fail("not refused: %s (%d instructions)" % (expr[:40], len(op)))


# ---------------------------------------------------------------------------------------------------- malformed programs
def _good():
    """energy theta*a + g, derivative a: one parameter, one global"""
    op = [OP["GLOBAL"], OP["PARAM"], OP["THETA"], OP["MUL"], OP["ADD"], OP["PARAM"]]
    return [0, 5, 6], op, [0, 0, 0, 0, 0, 0], [0.0]*6


def _refused(start, op, arg, imm, stride=1, nglobals=1):
    value, err = probe(start, op, arg, imm, stride, nglobals, 0, 0.5, [2.0], [0.25])
    assert value is None
    return err


def test_a_well_formed_program_runs():
    start, op, arg, imm = _good()
    assert probe(start, op, arg, imm, 1, 1, 0, 0.5, [2.0], [0.25])[0] == 0.5*2.0 + 0.25
    assert probe(start, op, arg, imm, 1, 1, 1, 0.5, [2.0], [0.25])[0] == 2.0


@pytest.mark.parametrize("case,match", [
    ("opcode", "unknown opcode"), ("negative opcode", "unknown opcode"), ("param", "parameter index"),
    ("global", "global parameter index"), ("underflow", "underflow"), ("leftover", "exactly one value"),
    ("deep", "deeper than 16"), ("empty", "empty program"), ("start", "prog_start"), ("stride", "16 parameters"),
])
def test_malformed_programs_are_refused(case, match):
    start, op, arg, imm = _good()
    stride, nglobals = 1, 1
    if case == "opcode":
        op[3] = 42
    elif case == "negative opcode":
        op[3] = -1
    elif case == "param":
        arg[1] = 1
    elif case == "global":
        arg[0] = 1
    elif case == "underflow":
        op, start = [OP["THETA"], OP["ADD"], OP["PARAM"]], [0, 2, 3]
    elif case == "leftover":
        op, start = [OP["THETA"], OP["THETA"], OP["PARAM"]], [0, 2, 3]
    elif case == "deep":
        op = [OP["THETA"]]*17 + [OP["ADD"]]*16 + [OP["PARAM"]]
        start = [0, 33, 34]
    elif case == "empty":
        start = [0, 0, 6]
    elif case == "start":
        start = [0, 6, 5]
    elif case == "stride":
        stride = 17
    arg = (arg + [0]*len(op))[:len(op)]
    imm = [0.0]*len(op)
    assert match in _refused(start, op, arg, imm, stride, nglobals)
