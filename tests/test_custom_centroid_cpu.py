"""CPU tests of custom centroid bonds: the plugin's translator makes for a centroid expression in g1..gN exactly the programs
of the compound-bond expression in p1..pN; the double-precision yardstick (group centres from computeNormalizedWeights'
weights, the compound probe at the centres, forces spread with the weights) against the live Reference platform's
CustomCentroidBondForce; the limits validateSystem refuses."""
import re
import numpy as np
import pytest
import centroid_harness as H

pytestmark = pytest.mark.skipif(not H.available(), reason="oracle/_ref (the built reference and the test C APIs) is absent")

EXPRESSIONS = [
    ("0.5*k*(distance(g1,g2)-r0)^2", 2, ("k", "r0")),
    ("k*(angle(g1,g2,g3)-a0)^2 + distance(g1,g3)", 3, ("k", "a0")),
    ("k*(1+cos(2*dihedral(g1,g2,g3,g4)-a0))", 4, ("k", "a0")),
    ("k*pointdistance(x1,y1,z1,x2,y2,z2)^2 + pointangle(x1,y1,z1,x2,y2,z2,x3,y3,z3)", 3, ("k",)),
    ("pointdihedral(x1,y1,z1,x2,y2,z2,x3,y3,z3,x4,y4,z4)*k", 4, ("k",)),
    ("0.5*k*step(dr)*dr^2; dr = pointdistance(x1, y1, z1, x0, y0, z0) - rflat", 1, ("k", "x0", "y0", "z0", "rflat")),
]


@pytest.mark.parametrize("energy,n,params", EXPRESSIONS, ids=["distance", "angle", "dihedral", "point", "pointdihedral", "flat"])
def test_centroid_programs_are_the_compound_programs(energy, n, params):
    centroid = H.translate(H.CENTROID, energy, params, ("lam",), n)
    compound = H.translate(H.COMPOUND, re.sub(r"\bg(\d)\b", r"p\1", energy), params, ("lam",), n)
    assert len(centroid[3]) == 2 + 3*n
    for a, b in zip(centroid, compound):
        assert np.array_equal(a, b)


def _system(periodic=False, seed=3, n=14):
    from openmm_b200 import systems
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 2.0, (n, 3))
    if periodic:
        x[: n//2] += [2.5, -1.5, 0.7]          # outside the primary cell
    return systems.SystemDesc(masses=rng.uniform(1.0, 16.0, n), charges=np.zeros(n), sigmas=np.full(n, 0.3), epsilons=np.zeros(n),
                              positions=x, box=np.diag([2.2, 2.4, 2.6]) if periodic else None,
                              method=systems.NB_CUTOFF_PERIODIC if periodic else systems.NB_NOCUTOFF, cutoff=1.0, use_dispersion=False)


def _restrained(case):
    from openmm_b200 import systems
    periodic = case == "periodic"
    d = _system(periodic)
    a, b, c = [0, 1, 2, 3], [4, 5, 6, 7, 8], [9, 10, 11, 12, 13]
    weights = None
    if case in ("custom", "periodic"):
        weights = [[1.0, 2.0, 0.5, 3.0], [1.0, 0.0, 1.0, 4.0, 2.0]]
    d = systems.with_centroid_restraint(d, [a, b], systems.COM_DISTANCE_RESTRAINT, [[300.0, 0.4]], ("k", "r0"), weights=weights,
                                        periodic=periodic)
    if case == "overlap":
        # overlapping groups, one group in several bonds, a one-group flat-bottom restraint beside
        d = systems.with_centroid_restraint(d, [[3, 4, 5], c, [0, 9]], "k*(angle(g1,g2,g3)-a0)^2", [[40.0, 1.2], [25.0, 0.8]], ("k", "a0"),
                                            bonds=[[0, 1, 2], [2, 0, 1]])
        d = systems.with_centroid_restraint(d, [c], systems.FLAT_BOTTOM_RESTRAINT, [[500.0, 0.9, 1.1, 0.8, 0.2]],
                                            ("k", "x0", "y0", "z0", "rflat"))
    return H.compiled(d)


@pytest.mark.parametrize("case", ["mass", "custom", "overlap", "periodic"])
def test_yardstick_matches_the_reference_platform(case):
    d = _restrained(case)
    ref = H.Simulation(d, "Reference", force_groups={"custom_centroid": 5})
    w = ref.normalized_weights(0)          # every centroid force of the harness holds every group
    assert np.abs(w - d.ccentroid_group_weights).max() <= 1e-15
    fr, er = ref.forces_energy(1 << 5)
    e, f = H.centroid_yardstick(d, d.positions, weights=w)
    assert abs(e - er) <= 1e-10*abs(er) and abs(er) > 1e-3, (e, er)
    assert np.abs(f - fr).max() <= 1e-10*np.abs(fr).max(), np.abs(f - fr).max()
    assert np.abs(fr).max() > 1.0


def _small_centroid(energy, groups_per_bond, names=(), ngroups=None):
    from openmm_b200 import systems
    ngroups = groups_per_bond if ngroups is None else ngroups
    d = _system(n=max(2, ngroups))
    return systems.with_centroid_restraint(d, [[g] for g in range(ngroups)], energy, np.zeros((1, len(names))), names,
                                           bonds=[list(range(groups_per_bond))])


def test_limits_are_refused_as_unsupported():
    nine = "+".join("x%d" % i for i in range(1, 10))
    with pytest.raises(H.Refused, match="CustomCentroidBondForce with more than 8 groups per bond"):
        H.translate(H.CENTROID, nine, nparticles=9)
    names = tuple("c%d" % i for i in range(17))
    with pytest.raises(H.Refused, match="CustomCentroidBondForce with more than 16 per-bond parameters"):
        H.translate(H.CENTROID, "distance(g1,g2)*(" + "+".join(names) + ")", names, nparticles=2)
    with pytest.raises(H.Refused, match="tabulated functions in a CustomCentroidBondForce"):
        H.translate(H.CENTROID, "fn(distance(g1,g2))", nparticles=2, tabulated=True)
    with pytest.raises(ValueError, match="Unknown variable"):
        H.translate(H.CENTROID, "1+none", nparticles=2)

