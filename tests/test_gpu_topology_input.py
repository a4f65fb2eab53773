"""GPU tests of the input checks of the bonded-topology calls: the set_* call that receives an atom index outside
[0, natoms), a negative count or a CMAP map index out of range refuses it, and b200md_last_error names the term class.
No context here computes, and only the last test finalizes one (with valid terms), so no kernel ever sees a refused index."""
import ctypes as C
import pytest
from openmm_b200 import _lib

pytestmark = pytest.mark.gpu
NATOMS = 8
# term class (as the error message names it) -> (set_* call, atoms per term)
CLASSES = {"exception": ("set_exceptions", 2), "bond": ("set_bonds", 2), "angle": ("set_angles", 3),
           "periodic torsion": ("set_torsions", 4), "RB torsion": ("set_rb_torsions", 4), "CMAP torsion": ("set_cmap", 8)}


def _ints(v):
    return (C.c_int*len(v))(*v)


def _dbls(v):
    return (C.c_double*len(v))(*v)


def _set(L, h, cls, n, terms, cmap_map=0):
    """the set_* call of `cls` with count n and the atoms of `terms` (one tuple per term; at least one, whatever n is)"""
    k = len(terms)
    col = [_ints([t[j] for t in terms]) for j in range(len(terms[0]))]
    d = _dbls([1.0]*k)
    if cls == "exception":
        return L.b200md_set_exceptions(h, n, col[0], col[1], d, d, d)
    if cls == "bond":
        return L.b200md_set_bonds(h, n, col[0], col[1], d, d)
    if cls == "angle":
        return L.b200md_set_angles(h, n, col[0], col[1], col[2], d, d)
    if cls == "periodic torsion":
        return L.b200md_set_torsions(h, n, col[0], col[1], col[2], col[3], _ints([3]*k), d, d)
    if cls == "RB torsion":
        return L.b200md_set_rb_torsions(h, n, col[0], col[1], col[2], col[3], _dbls([0.5]*6*k))
    # one 2 x 2 map: 4 patches of 16 coefficients
    return L.b200md_set_cmap(h, 1, _ints([2]), _dbls([0.0]*64), n, _ints([cmap_map]*k), _ints([a for t in terms for a in t]))


@pytest.fixture
def ctx():
    L = _lib.load()
    h = C.c_void_p()
    assert L.b200md_create(C.byref(h), 0, NATOMS) == 0, L.b200md_last_error(None)
    yield L, h
    L.b200md_destroy(h)


def _valid(cls, n=3):
    arity = CLASSES[cls][1]
    return [tuple((t + j) % NATOMS for j in range(arity)) for t in range(n)]


@pytest.mark.parametrize("cls", list(CLASSES))
def test_valid_terms_are_accepted(ctx, cls):
    L, h = ctx
    assert _set(L, h, cls, 3, _valid(cls)) == 0, L.b200md_last_error(h)
    assert _set(L, h, cls, 0, _valid(cls, 1)) == 0, L.b200md_last_error(h)


@pytest.mark.parametrize("bad", [NATOMS, -1])
@pytest.mark.parametrize("cls", list(CLASSES))
def test_atom_index_out_of_range_is_refused(ctx, cls, bad):
    """every atom position of a term, in the last of three terms"""
    L, h = ctx
    for pos in range(CLASSES[cls][1]):
        terms = _valid(cls)
        terms[-1] = tuple(bad if j == pos else a for j, a in enumerate(terms[-1]))
        assert _set(L, h, cls, 3, terms) == -1, (cls, pos)
        assert L.b200md_last_error(h) == (cls + ": atom index out of range").encode()


@pytest.mark.parametrize("cls", list(CLASSES))
def test_negative_count_is_refused(ctx, cls):
    L, h = ctx
    assert _set(L, h, cls, -1, _valid(cls, 1)) == -1
    assert L.b200md_last_error(h) == ("%s: negative count" % CLASSES[cls][0]).encode()


@pytest.mark.parametrize("bad", [1, -1])
def test_cmap_map_index_out_of_range_is_refused(ctx, bad):
    L, h = ctx
    assert _set(L, h, "CMAP torsion", 3, _valid("CMAP torsion"), cmap_map=bad) == -1
    assert L.b200md_last_error(h) == b"CMAP torsion: map index out of range"


def test_finalize_after_a_refused_box_succeeds(ctx):
    """finalize refuses a periodic box under twice the cutoff and leaves the context unfinalized; with the box fixed, the
    next finalize succeeds.  Bonds are set, the other term classes are empty: the force groups are checked against the
    terms at every finalize, and padding an empty class's groups for the device must not change that check's input."""
    from openmm_b200 import systems
    L, h = ctx
    assert _set(L, h, "bond", 3, _valid("bond")) == 0
    desc = _lib.NonbondedDesc(method=systems.NB_CUTOFF_PERIODIC, cutoff=1.0, rf_dielectric=78.3)
    q, sig, eps = _dbls([0.0]*NATOMS), _dbls([0.3]*NATOMS), _dbls([0.5]*NATOMS)
    assert L.b200md_set_nonbonded(h, C.byref(desc), q, sig, eps) == 0, L.b200md_last_error(h)

    def box(edge):
        return L.b200md_set_box(h, _dbls([edge, 0, 0]), _dbls([0, edge, 0]), _dbls([0, 0, edge]))
    assert box(1.5) == 0
    assert L.b200md_finalize(h) == -1
    assert b"less than twice the nonbonded cutoff" in L.b200md_last_error(h)
    assert box(3.0) == 0
    assert L.b200md_finalize(h) == 0, L.b200md_last_error(h)
