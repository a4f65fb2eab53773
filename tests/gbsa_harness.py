"""Test harness of the generalized Born (GBSAOBCForce) tests: the systems they use, a double-precision restatement of OBC II +
ACE in numpy (the yardstick of the engine-level tests), and the reference's Simulation with a GBSAOBCForce added, over
oracle/_ref/tests/libgbsa_capi.so (plugin/tests/gbsa_capi.cpp).

The restatement follows the closed forms of gbsa.cu's header (Onufriev, Bashford and Case, Proteins 55:383, 2004; ACE of
Schaefer, Bartels and Karplus, 1998): Born sums over every pair within the cutoff, excluded pairs included; the GB pair energy
over i <= j with the self term at half weight and, with a cutoff, shifted by -f q_i q_j/cutoff; forces as the analytic
gradient the Reference platform evaluates."""
import ctypes as C
import os

import numpy as np

from openmm_b200 import systems
from oracle import omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "oracle", "_ref", "tests", "libgbsa_capi.so")
FIXTURE = os.path.join(ROOT, "tests", "golden", "dhfr_gbsa.npz")
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_gbsa.npz")
ONE_4PI_EPS0 = 138.93545764438198
OFFSET, PROBE, ALPHA, BETA, GAMMA = 0.009, 0.14, 1.0, 0.8, 4.85
GB_GROUP = 3
_lib = None


def available():
    return os.path.exists(LIB) and omm.available()


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(LIB)
        D, I, P = C.POINTER(C.c_double), C.c_int, C.c_void_p
        L.gbc_add_force.argtypes = [P, I, D, D, D, I, C.c_double, C.c_double, C.c_double, C.c_double, I]
        L.gbc_add_force.restype = I
        L.gbc_update.argtypes = [P, I, P, I, D, D, D]
        L.gbc_update.restype = I
        L.gbc_last_error.restype = C.c_char_p
        L.gbc_default_platform.argtypes = [P]
        L.gbc_default_platform.restype = C.c_char_p
        _lib = L
    return _lib


def _dp(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


# ---------------------------------------------------------------- systems
def dhfr_gbsa(method=systems.NB_CUTOFF_NONPERIODIC):
    """The DHFR implicit-solvent fixture (amber99sb + amber99_obc, 5dfr_minimized.pdb, HBonds, CutoffNonPeriodic 2 nm); with
    method NB_NOCUTOFF both forces switch to NoCutoff."""
    d = systems.SystemDesc.load(FIXTURE)
    if method == systems.NB_NOCUTOFF:
        d.method = d.gb_method = systems.NB_NOCUTOFF
    return d


def without_gbsa(desc):
    import copy
    d = copy.copy(desc)
    d.gb_charges, d.gb_radii, d.gb_scales = np.zeros(0), np.zeros(0), np.zeros(0)
    return d


def hello_nacl():
    """The six ions of the reference's HelloSodiumChloride example (NoCutoff, GBSA with dielectrics 2 and 80)."""
    na = (22.99, 1.0, 1.8680, 0.00277, 1.992, 0.8)
    cl = (35.45, -1.0, 2.4700, 0.1000, 1.735, 0.8)
    ions = [na, cl, na, cl, na, cl]
    pos = np.array([[8, 0, 0], [-8, 0, 0], [0, 9, 0], [0, -9, 0], [0, 0, -10], [0, 0, 10]], dtype=float)*0.1
    sigma_per_radius = 2.0/2.0**(1.0/6.0)
    d = systems.SystemDesc(masses=np.array([a[0] for a in ions]), charges=np.array([a[1] for a in ions]),
                           sigmas=np.array([a[2]*0.1*sigma_per_radius for a in ions]), epsilons=np.array([a[3]*4.184 for a in ions]),
                           positions=pos, box=None, method=systems.NB_NOCUTOFF, cutoff=1.0, use_dispersion=False, name="hello_nacl")
    d.gb_charges = d.charges.copy()
    d.gb_radii = np.array([a[4]*0.1 for a in ions])
    d.gb_scales = np.array([a[5] for a in ions])
    d.gb_method = systems.NB_NOCUTOFF
    d.gb_solute_dielectric, d.gb_solvent_dielectric = 2.0, 80.0
    return d


def ion_box(n=400, edge=3.2, cutoff=1.2, method=systems.NB_CUTOFF_PERIODIC, seed=11, box=None):
    """n ions of alternating charge +-1 on a jittered lattice in a cubic box of edge `edge`, or of the cell `box` (rows a,
    b, c; reduced form) when given; GBSA radii 0.15-0.2 nm.  Periodic methods keep the box, NB_NOCUTOFF and
    NB_CUTOFF_NONPERIODIC drop it.  The GBSAOBCForce takes CutoffPeriodic for PME."""
    rng = np.random.default_rng(seed)
    m = int(np.ceil(n**(1/3)))
    g = np.stack(np.meshgrid(*[np.arange(m)]*3, indexing="ij"), -1).reshape(-1, 3)[:n]
    if box is None:
        pos = (g + 0.5 + 0.25*rng.uniform(-1, 1, (n, 3)))*(edge/m)
        box = np.eye(3)*edge
    else:
        box = np.asarray(box, dtype=np.float64)
        pos = ((g + 0.5 + 0.25*rng.uniform(-1, 1, (n, 3)))/m) @ box
    q = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    periodic = method in (systems.NB_CUTOFF_PERIODIC, systems.NB_PME)
    d = systems.SystemDesc(masses=np.full(n, 30.0), charges=q, sigmas=np.full(n, 0.3), epsilons=np.full(n, 0.4), positions=pos,
                           box=box if periodic else None, method=method, cutoff=cutoff, rf_dielectric=1.0,
                           use_dispersion=False, name="ion_box")
    d.gb_charges = q.copy()
    d.gb_radii = rng.uniform(0.15, 0.2, n)
    d.gb_scales = rng.uniform(0.7, 0.9, n)
    d.gb_method = systems.NB_CUTOFF_PERIODIC if periodic else method
    return d


# the edges of OpenMM's reduced form (a = 3 nm, b.x = +-a/2, c.x = -+a/2, c.y = +-b/2), as tests/test_gpu_oracle_edges.py
TRICLINIC_LIMITS = {"pmp": (1.5, -1.5, 1.5), "mpm": (-1.5, 1.5, -1.5)}


def triclinic_ion_box(sign):
    """400 ions in the reduced-form limit cell `sign` (a key of TRICLINIC_LIMITS), CutoffPeriodic at 0.49 times the
    smallest cell width (1.09 nm of 2.23): every pair within the cutoff has one image that the single-pass reduction of
    ReferenceForce::getDeltaRPeriodic finds"""
    bx, cx, cy = TRICLINIC_LIMITS[sign]
    box = np.array([[3.0, 0, 0], [bx, 3.0, 0], [cx, cy, 3.0]])
    a, b, c = box
    v = abs(np.dot(a, np.cross(b, c)))
    width = min(v/np.linalg.norm(np.cross(b, c)), v/np.linalg.norm(np.cross(c, a)), v/np.linalg.norm(np.cross(a, b)))
    d = ion_box(cutoff=round(0.49*width, 2), box=box, seed=12)
    d.name = "ion_box_tri_" + sign
    return d


def golden_cases():
    """The cases of tests/golden/reference_gbsa.npz (make_golden_gbsa.py), by name"""
    custom = ion_box(method=systems.NB_NOCUTOFF)
    custom.gb_surface_area_energy, custom.gb_solute_dielectric, custom.gb_solvent_dielectric = 0.0, 4.0, 40.0
    return {"dhfr_nocutoff": dhfr_gbsa(systems.NB_NOCUTOFF), "dhfr_cutoff": dhfr_gbsa(), "hello_nacl": hello_nacl(),
            "ion_box": ion_box(), "ion_box_custom": custom,
            "ion_box_tri_pmp": triclinic_ion_box("pmp"), "ion_box_tri_mpm": triclinic_ion_box("mpm")}


# ---------------------------------------------------------------- the restatement
def _displacements(x, rows, box, periodic):
    """x[j] - x[i] for i in rows, all j; minimum image as ReferenceForce::getDeltaRPeriodic (c, b, a order)."""
    d = x[None, :, :] - x[rows, None, :]
    if periodic:
        a, b, c = box
        k = np.floor(d[..., 2]/c[2] + 0.5)
        d -= k[..., None]*c
        k = np.floor(d[..., 1]/b[1] + 0.5)
        d -= k[..., None]*b
        k = np.floor(d[..., 0]/a[0] + 0.5)
        d -= k[..., None]*a
    return d


def _integral(r, rho, sr):
    with np.errstate(divide="ignore", invalid="ignore"):
        active = rho < r + sr
        l = 1.0/np.maximum(rho, np.abs(r - sr))
        u = 1.0/(r + sr)
        t = l - u + 0.25*r*(u*u - l*l) + 0.5/r*np.log(u/l) + 0.25*sr*sr/r*(l*l - u*u)
        t = t + np.where(rho < sr - r, 2.0*(1.0/rho - l), 0.0)
        d = 0.125*(1.0 + sr*sr/(r*r))*(l*l - u*u) + 0.25*np.log(u/l)/(r*r)
    return np.where(active, t, 0.0), np.where(active, d, 0.0)


def obc_forces_energy(desc, x=None, chunk=256):
    """Energy (kJ/mol) and forces (kJ/mol/nm) of desc's GBSAOBCForce alone at positions x, in double precision."""
    x = np.asarray(desc.positions if x is None else x, dtype=np.float64)
    n = len(x)
    q, R, s = (np.asarray(a, dtype=np.float64) for a in (desc.gb_charges, desc.gb_radii, desc.gb_scales))
    rho = R - OFFSET
    sr = s*rho
    use_cutoff = desc.gb_method != systems.NB_NOCUTOFF
    periodic = desc.gb_method == systems.NB_CUTOFF_PERIODIC
    box = None if desc.box is None else np.asarray(desc.box, dtype=np.float64)
    eps_in, eps_out = desc.gb_solute_dielectric, desc.gb_solvent_dielectric
    pf = -ONE_4PI_EPS0*(1.0/eps_in - 1.0/eps_out) if eps_in != 0.0 and eps_out != 0.0 else 0.0

    def blocks():
        for i0 in range(0, n, chunk):
            rows = np.arange(i0, min(n, i0 + chunk))
            d = _displacements(x, rows, box, periodic)
            r = np.sqrt((d*d).sum(-1))
            mask = rows[:, None] != np.arange(n)[None, :]
            if use_cutoff:
                mask &= r <= desc.cutoff
            yield rows, d, np.where(mask, r, 1.0), mask

    S = np.zeros(n)
    for rows, d, r, mask in blocks():
        S[rows] = np.where(mask, _integral(r, rho[rows, None], sr[None, :])[0], 0.0).sum(1)
    psi = 0.5*rho*S
    T = np.tanh(psi*(ALPHA + psi*(-BETA + GAMMA*psi)))
    B = 1.0/(1.0/rho - T/R)
    chain = rho*(ALPHA - 2.0*BETA*psi + 3.0*GAMMA*psi*psi)*(1.0 - T*T)/R
    sa = np.where(B > 0.0, 4.0*np.pi*desc.gb_surface_area_energy*(R + PROBE)**2*(R/B)**6, 0.0)
    self_g = pf*q*q/B
    energy = sa.sum() + 0.5*self_g.sum()
    dEdB = -6.0*sa/B - 0.5*self_g/B
    f = np.zeros((n, 3))
    shift = 1.0/desc.cutoff if use_cutoff else 0.0
    for rows, d, r, mask in blocks():
        r2 = r*r
        a2 = B[rows, None]*B[None, :]
        D = 0.25*r2/a2
        ex = np.exp(-D)
        den2 = r2 + a2*ex
        qq = pf*q[rows, None]*q[None, :]
        G = qq/np.sqrt(den2)
        dGdr = np.where(mask, -G*(1.0 - 0.25*ex)/den2, 0.0)
        dGda2 = np.where(mask, -0.5*G*ex*(1.0 + D)/den2, 0.0)
        energy += 0.5*np.where(mask, G - qq*shift, 0.0).sum()
        dEdB[rows] += (dGda2*B[None, :]).sum(1)
        f[rows] += (d*dGdr[..., None]).sum(1)
    bf = dEdB*B*B*chain
    for rows, d, r, mask in blocks():
        dij = _integral(r, rho[rows, None], sr[None, :])[1]
        dji = _integral(r, rho[None, :], sr[rows, None])[1]
        de = np.where(mask, (bf[rows, None]*dij + bf[None, :]*dji)/r, 0.0)
        f[rows] -= (d*de[..., None]).sum(1)
    return f, float(energy)


# ---------------------------------------------------------------- the reference
class Simulation(omm.Simulation):
    """oracle.omm.Simulation plus desc's GBSAOBCForce (when it has one) in force group GB_GROUP; everything else stays in
    group 0.  The GBSAOBCForce's method is desc.gb_method and its cutoff desc.cutoff."""

    def add_forces(self):
        super().add_forces()
        d = self.desc
        self.gb_index = None
        if len(d.gb_charges):
            self.gb_index = lib().gbc_add_force(self.sys, len(d.gb_charges), _dp(d.gb_charges), _dp(d.gb_radii), _dp(d.gb_scales),
                                                int(d.gb_method), float(d.cutoff), float(d.gb_solute_dielectric),
                                                float(d.gb_solvent_dielectric), float(d.gb_surface_area_energy), GB_GROUP)
            if self.gb_index < 0:
                raise RuntimeError(lib().gbc_last_error().decode())

    def default_platform(self):
        """the platform a Context of this System gets when none is named"""
        return lib().gbc_default_platform(self.sys).decode()

    def update_gbsa(self, charges, radii, scales):
        if lib().gbc_update(self.sys, self.gb_index, self.ctx, len(charges), _dp(charges), _dp(radii), _dp(scales)) != 0:
            raise RuntimeError(lib().gbc_last_error().decode())


def gb_only(sim):
    """(forces, energy) of the GBSAOBCForce group of a Simulation"""
    return sim.forces_energy(groups=1 << GB_GROUP)


def force_error(f, ref):
    """max over atoms of max|df| / max(1, |f_ref|)"""
    return float((np.abs(f - ref).max(axis=1)/np.maximum(1.0, np.linalg.norm(ref, axis=1))).max())
