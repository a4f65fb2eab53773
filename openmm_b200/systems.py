"""Benchmark / test systems as plain numpy descriptions (consumed by Engine and by the oracle harness alike).

Builders follow SURVEY.md 8(d): S1 = TIP3P water lattice (the DHFR-sized proxy), LJ fluids, random ion boxes.
PME parameter selection restates NonbondedForceImpl::calcPMEParameters (openmmapi/src/NonbondedForceImpl.cpp:160-184)
and the dispersion coefficient NonbondedForceImpl::calcDispersionCorrection (:236-310) -- the OpenMM plugin calls the
reference's own static helpers instead; these restatements exist so that the Python harness has no OpenMM dependency.
"""
from dataclasses import dataclass, field
import math
import ctypes
import numpy as np

NB_NOCUTOFF, NB_CUTOFF_NONPERIODIC, NB_CUTOFF_PERIODIC, NB_EWALD, NB_PME, NB_LJPME = range(6)
INT_VERLET, INT_LANGEVIN, INT_LANGEVIN_MIDDLE = range(3)


def _i(n=0):
    return np.zeros(n, dtype=np.int32)


def _d(n=0):
    return np.zeros(n, dtype=np.float64)


@dataclass
class SystemDesc:
    masses: np.ndarray
    charges: np.ndarray
    sigmas: np.ndarray
    epsilons: np.ndarray
    positions: np.ndarray                      # [N,3] nm
    box: np.ndarray = None                     # [3,3] rows a,b,c (reduced form) or None
    method: int = NB_PME
    cutoff: float = 1.0
    ewald_tol: float = 5e-4
    use_switch: bool = False
    switch_distance: float = 0.0
    rf_dielectric: float = 78.3
    use_dispersion: bool = True
    pme_alpha: float = 0.0                     # 0 -> derive from tolerance
    pme_grid: tuple = (0, 0, 0)
    exc_i: np.ndarray = field(default_factory=_i)
    exc_j: np.ndarray = field(default_factory=_i)
    exc_qq: np.ndarray = field(default_factory=_d)
    exc_sigma: np.ndarray = field(default_factory=_d)
    exc_eps: np.ndarray = field(default_factory=_d)
    bond_i: np.ndarray = field(default_factory=_i)
    bond_j: np.ndarray = field(default_factory=_i)
    bond_r0: np.ndarray = field(default_factory=_d)
    bond_k: np.ndarray = field(default_factory=_d)
    angle_i: np.ndarray = field(default_factory=_i)
    angle_j: np.ndarray = field(default_factory=_i)
    angle_k: np.ndarray = field(default_factory=_i)
    angle_t0: np.ndarray = field(default_factory=_d)
    angle_kk: np.ndarray = field(default_factory=_d)
    tor_i: np.ndarray = field(default_factory=_i)
    tor_j: np.ndarray = field(default_factory=_i)
    tor_k: np.ndarray = field(default_factory=_i)
    tor_l: np.ndarray = field(default_factory=_i)
    tor_n: np.ndarray = field(default_factory=_i)
    tor_phase: np.ndarray = field(default_factory=_d)
    tor_kk: np.ndarray = field(default_factory=_d)
    rb_i: np.ndarray = field(default_factory=_i)          # RBTorsionForce
    rb_j: np.ndarray = field(default_factory=_i)
    rb_k: np.ndarray = field(default_factory=_i)
    rb_l: np.ndarray = field(default_factory=_i)
    rb_c: np.ndarray = field(default_factory=lambda: np.zeros((0, 6)))       # [n,6] c0..c5, kJ/mol
    cmap_size: np.ndarray = field(default_factory=_i)     # CMAPTorsionForce: [nmaps] map sizes
    cmap_coeff: np.ndarray = field(default_factory=_d)    # [sum size^2, 16] bicubic coefficients (CMAPTorsionForceImpl::calcMapDerivatives)
    cmap_energy: np.ndarray = field(default_factory=_d)   # [sum size^2] map energies, kJ/mol (what a CMAPTorsionForce is given)
    cmap_map: np.ndarray = field(default_factory=_i)      # [n] map of each term
    cmap_atoms: np.ndarray = field(default_factory=lambda: np.zeros((0, 8), dtype=np.int32))   # [n,8] the two dihedrals
    # CustomTorsionForce: per expression p its energy (a Lepton expression of theta, the per-torsion parameters
    # custom_param_names[p] and the global parameters custom_global_names), and per term its expression, atoms and parameters.
    # custom_prog_start / op / arg / imm are the compiled programs b200md_set_custom_torsions takes (program 2p = energy of
    # expression p, 2p+1 = its dE/dtheta); they come from the plugin's translator (plugin/custom_translate.h).
    custom_energy: tuple = ()
    custom_param_names: tuple = ()                        # per expression: the names of its per-torsion parameters
    custom_global_names: tuple = ()                       # global slot s <- name s
    custom_global_values: np.ndarray = field(default_factory=_d)
    custom_prog: np.ndarray = field(default_factory=_i)   # [n] expression of each term
    custom_atoms: np.ndarray = field(default_factory=lambda: np.zeros((0, 4), dtype=np.int32))
    custom_params: np.ndarray = field(default_factory=lambda: np.zeros((0, 0)))   # [n, param_stride]
    custom_prog_start: np.ndarray = field(default_factory=_i)
    custom_op: np.ndarray = field(default_factory=_i)
    custom_arg: np.ndarray = field(default_factory=_i)
    custom_imm: np.ndarray = field(default_factory=_d)
    con_i: np.ndarray = field(default_factory=_i)
    con_j: np.ndarray = field(default_factory=_i)
    con_d: np.ndarray = field(default_factory=_d)
    cm_frequency: int = 0
    name: str = "system"

    @property
    def natoms(self):
        return len(self.masses)

    def pme_parameters(self, friendly=True):
        """(alpha, nx, ny, nz).  friendly=True rounds each dimension up to the next size the bespoke FFT factors
        into radices <= 16 (as the reference CUDA platform rounds to 2,3,5,7-smooth sizes, CudaKernels.cpp:698-700)."""
        if self.pme_alpha != 0.0:
            return self.pme_alpha, *self.pme_grid
        tol = self.ewald_tol
        alpha = (1.0/self.cutoff)*math.sqrt(-math.log(2.0*tol))
        dims = []
        for d in range(3):
            n = max(int(math.ceil(2*alpha*self.box[d][d]/(3*tol**0.2))), 6)
            if friendly:
                n = next_fft_size(n)
            dims.append(n)
        return alpha, dims[0], dims[1], dims[2]

    def dispersion_coefficient(self):
        if not self.use_dispersion or self.method in (NB_NOCUTOFF, NB_CUTOFF_NONPERIODIC):
            return 0.0
        return dispersion_coefficient(self.sigmas, self.epsilons, self.cutoff, self.use_switch, self.switch_distance)

    def molecules(self):
        """The molecules a barostat moves as rigid groups, as ContextImpl::getMolecules() forms them: connected components of
        the constraints and the HarmonicBondForce bonds (ContextImpl.cpp:351-383; angles, torsions and exceptions do not
        join molecules).  Ordered by their lowest atom, atoms ascending (ContextImpl::findMolecules)."""
        n = self.natoms
        parent = np.arange(n)

        def find(x):
            while parent[x] != x:
                parent[x] = parent[parent[x]]
                x = parent[x]
            return x
        for i, j in zip(np.concatenate([self.con_i, self.bond_i]).tolist(), np.concatenate([self.con_j, self.bond_j]).tolist()):
            a, b = find(i), find(j)
            if a != b:
                parent[max(a, b)] = min(a, b)
        groups = {}
        for i in range(n):
            groups.setdefault(find(i), []).append(i)
        return [groups[r] for r in sorted(groups)]

    def rounded(self):
        """Same system with fp32-representable positions: the identical inputs both the fp32 device path and the
        double-precision oracle are given in parity tests."""
        import copy
        d = copy.copy(self)
        d.positions = np.asarray(self.positions, dtype=np.float32).astype(np.float64)
        return d

    def save(self, path):
        d = {k: (np.asarray(v) if v is not None else np.zeros(0)) for k, v in self.__dict__.items()
             if not isinstance(v, str) and k != "custom_param_names"}
        width = max([len(p) for p in self.custom_param_names] + [0])
        rows = [list(p) + [""]*(width - len(p)) for p in self.custom_param_names]
        d["custom_param_names"] = np.array(rows, dtype=str).reshape(len(rows), width)
        d["name"] = np.array(self.name)
        np.savez_compressed(path, **d)

    @staticmethod
    def load(path):
        z = np.load(path, allow_pickle=False)
        kw = {}
        for k in z.files:
            v = z[k]
            if k == "name":
                kw[k] = str(v)
            elif k in ("custom_energy", "custom_global_names"):
                kw[k] = tuple(str(x) for x in v)
            elif k == "custom_param_names":
                kw[k] = tuple(tuple(str(y) for y in x if str(y)) for x in v)
            elif k == "box":
                kw[k] = v if v.size == 9 else None
            elif k == "pme_grid":
                kw[k] = tuple(int(x) for x in v)
            elif v.ndim == 0:
                kw[k] = v.item()
            else:
                kw[k] = v
        return SystemDesc(**kw)


def periodic_to_rb(desc):
    """The same System with every periodic torsion k (1 + cos(n phi - phase)), n <= 3 and phase 0 or pi, written as an exactly
    equal Ryckaert-Bellemans torsion sum_m c_m cos^m psi, psi = phi - pi: cos(n phi) = T_n(cos phi) = (-1)^n T_n(cos psi)."""
    import copy
    cheb = {0: [1, 0, 0, 0], 1: [0, 1, 0, 0], 2: [-1, 0, 2, 0], 3: [0, -3, 0, 4]}
    n, ph, k = np.asarray(desc.tor_n), np.asarray(desc.tor_phase, dtype=np.float64), np.asarray(desc.tor_kk, dtype=np.float64)
    if len(n) and (n.max() > 3 or n.min() < 0):
        raise ValueError("periodic_to_rb: periodicity above 3")
    # force fields write pi with about 12 digits (3.14159265359): a phase that far from pi changes a force by ~1e-12 relative
    sign = np.where(np.abs(ph) < 1e-9, 1.0, np.where(np.abs(ph - math.pi) < 1e-9, -1.0, np.nan))
    if np.isnan(sign).any():
        raise ValueError("periodic_to_rb: a phase is neither 0 nor pi")
    c = np.zeros((len(n), 6))
    c[:, 0] = k
    for m in range(4):
        c[:, m] += k*sign*np.array([cheb[int(x)][m]*(-1)**int(x) for x in n])
    d = copy.copy(desc)
    d.rb_i, d.rb_j, d.rb_k, d.rb_l = (np.array(a, dtype=np.int32) for a in (desc.tor_i, desc.tor_j, desc.tor_k, desc.tor_l))
    d.rb_c = c
    d.tor_i, d.tor_j, d.tor_k, d.tor_l, d.tor_n, d.tor_phase, d.tor_kk = _i(), _i(), _i(), _i(), _i(), _d(), _d()
    return d


PERIODIC_CUSTOM = "k*(1+cos(n*theta-theta0))"
# CharmmPsfFile.createSystem's improper energy (app/charmmpsffile.py): harmonic in the angle's distance from theta0 across the
# +-pi seam; pi as that code writes it ('pi = %f')
CHARMM_IMPROPER = "k*min(dtheta, 2*pi-dtheta)^2; dtheta = abs(theta-theta0); pi = %f;" % math.pi


def _custom_only(desc, energy, param_names, prog, atoms, params, global_names=(), global_values=()):
    """desc with exactly these custom torsions (expressions not compiled yet)"""
    import copy
    d = copy.copy(desc)
    d.custom_energy, d.custom_param_names = tuple(energy), tuple(tuple(p) for p in param_names)
    d.custom_global_names, d.custom_global_values = tuple(global_names), np.asarray(global_values, dtype=np.float64)
    d.custom_prog = np.asarray(prog, dtype=np.int32)
    d.custom_atoms = np.asarray(atoms, dtype=np.int32).reshape(-1, 4)
    width = max([len(p) for p in d.custom_param_names] + [0])
    d.custom_params = np.asarray(params, dtype=np.float64).reshape(len(d.custom_prog), -1) if len(d.custom_prog) else np.zeros((0, width))
    d.custom_prog_start, d.custom_op, d.custom_arg, d.custom_imm = _i(), _i(), _i(), _d()
    return d


def periodic_to_custom(desc):
    """The same System with every periodic torsion k (1 + cos(n theta - theta0)) written as the CustomTorsionForce
    PERIODIC_CUSTOM with per-torsion parameters (k, n, theta0): the exact counterpart of periodic_to_rb."""
    atoms = np.stack([desc.tor_i, desc.tor_j, desc.tor_k, desc.tor_l], axis=1) if len(desc.tor_i) else np.zeros((0, 4))
    params = np.stack([desc.tor_kk, np.asarray(desc.tor_n, dtype=np.float64), desc.tor_phase], axis=1) if len(desc.tor_i) else np.zeros((0, 3))
    d = _custom_only(desc, [PERIODIC_CUSTOM], [("k", "n", "theta0")], np.zeros(len(desc.tor_i)), atoms, params)
    d.tor_i, d.tor_j, d.tor_k, d.tor_l, d.tor_n, d.tor_phase, d.tor_kk = _i(), _i(), _i(), _i(), _i(), _d(), _d()
    return d


def improper_centres(desc):
    """[n,4] impropers (centre, a, b, c) on every atom with exactly three bonded neighbours (bonds and constraints), the
    neighbours in ascending order; ordered by the centre."""
    nbr = [set() for _ in range(desc.natoms)]
    for i, j in zip(np.concatenate([desc.bond_i, desc.con_i]).tolist(), np.concatenate([desc.bond_j, desc.con_j]).tolist()):
        nbr[i].add(j)
        nbr[j].add(i)
    return np.array([[a] + sorted(nbr[a]) for a in range(desc.natoms) if len(nbr[a]) == 3], dtype=np.int32).reshape(-1, 4)


def with_charmm_impropers(desc, seed=1, k_range=(20.0, 800.0)):
    """desc plus one CHARMM improper (CHARMM_IMPROPER, per-torsion parameters k, theta0) per improper_centres quadruple, k
    uniform in k_range kJ/mol/rad^2 and theta0 at the current dihedral plus up to 0.3 rad, both from `seed`: the form
    CharmmPsfFile writes, with parameters that keep the terms near their minimum as force-field impropers are."""
    atoms = improper_centres(desc)
    rng = np.random.default_rng(seed)
    x = np.asarray(desc.positions, dtype=np.float64)
    theta = dihedrals(x, atoms, desc.box)
    k = rng.uniform(k_range[0], k_range[1], len(atoms))
    theta0 = np.mod(theta + rng.uniform(-0.3, 0.3, len(atoms)) + math.pi, 2*math.pi) - math.pi
    return _custom_only(desc, [CHARMM_IMPROPER], [("k", "theta0")], np.zeros(len(atoms)), atoms, np.stack([k, theta0], axis=1))


def dihedrals(x, atoms, box=None):
    """Dihedral angle in (-pi, pi] of every quadruple of atoms [n,4] at positions x, as ReferenceBondIxn measures it (the
    sign of the first difference vector against the second normal); minimum-image difference vectors when box is given."""
    def d(a, b):
        v = x[a] - x[b]
        if box is not None:
            bx = np.asarray(box, dtype=np.float64)
            for k in (2, 1, 0):
                v -= np.round(v[:, k:k+1]/bx[k, k])*bx[k]
        return v
    v0, v1, v2 = d(atoms[:, 0], atoms[:, 1]), d(atoms[:, 2], atoms[:, 1]), d(atoms[:, 2], atoms[:, 3])
    c0, c1 = np.cross(v0, v1), np.cross(v1, v2)
    cosang = np.clip(np.einsum("ij,ij->i", c0, c1)/np.sqrt(np.einsum("ij,ij->i", c0, c0)*np.einsum("ij,ij->i", c1, c1)), -1, 1)
    theta = np.arccos(cosang)
    return np.where(np.einsum("ij,ij->i", v0, c1) < 0, -theta, theta)


def backbone_cmap_atoms(desc):
    """[n,8] atoms of every backbone (phi, psi) pair: C(=O)-N-CA-C(=O)-N chains of the bond graph (bonds and constraints),
    with elements told apart by mass.  Ordered by the CA atom."""
    elem = np.select([np.abs(desc.masses - 12.011) < 0.1, np.abs(desc.masses - 14.007) < 0.1, np.abs(desc.masses - 15.999) < 0.1],
                     ["C", "N", "O"], "X")
    nbr = [set() for _ in range(desc.natoms)]
    for i, j in zip(np.concatenate([desc.bond_i, desc.con_i]).tolist(), np.concatenate([desc.bond_j, desc.con_j]).tolist()):
        nbr[i].add(j)
        nbr[j].add(i)
    carbonyl = [a for a in range(desc.natoms) if elem[a] == "C" and any(elem[o] == "O" and len(nbr[o]) == 1 for o in nbr[a])]
    is_co = np.zeros(desc.natoms, bool)
    is_co[carbonyl] = True
    out = []
    for c in carbonyl:                                  # C of residue i: ... N-CA-C(=O)-N(i+1)
        for ca in nbr[c]:
            if elem[ca] != "C" or is_co[ca]:
                continue
            for n in nbr[ca]:
                if elem[n] != "N":
                    continue
                for cp in nbr[n]:
                    if cp == ca or not is_co[cp]:
                        continue
                    for nn in nbr[c]:
                        if elem[nn] == "N":
                            out.append((cp, n, ca, c, n, ca, c, nn))
    out.sort(key=lambda t: t[2])
    return np.array(out, dtype=np.int32).reshape(-1, 8)


def with_cmap(desc, size, energy, coeff):
    """desc plus one CMAP term per backbone (phi, psi) pair (backbone_cmap_atoms), the maps assigned round robin.
    size [nmaps], energy [sum size^2] and coeff [sum size^2, 16] describe the maps."""
    import copy
    d = copy.copy(desc)
    d.cmap_atoms = backbone_cmap_atoms(desc)
    d.cmap_size = np.asarray(size, dtype=np.int32)
    d.cmap_energy = np.asarray(energy, dtype=np.float64)
    d.cmap_coeff = np.asarray(coeff, dtype=np.float64).reshape(-1, 16)
    d.cmap_map = (np.arange(len(d.cmap_atoms)) % len(d.cmap_size)).astype(np.int32)
    return d


def fft_size_ok(n):
    """True if n factors into radices <= 16 with at most 8 stages (the bespoke FFT's requirement, csrc/fft.cu)."""
    rem, stages = n, 0
    while rem > 1:
        for r in range(16, 1, -1):
            if rem % r == 0:
                rem //= r
                stages += 1
                break
        else:
            return False
    return stages <= 8


def next_fft_size(n):
    while not fft_size_ok(n):
        n += 1
    return n


def _eval_integral(r, rs, rc, sigma):
    # NonbondedForceImpl::evalIntegral (NonbondedForceImpl.cpp:200-234): indefinite integral of LJ x switch
    A = 1/(rc-rs)
    A2 = A*A
    A3 = A2*A
    sig2 = sigma*sigma
    sig6 = sig2*sig2*sig2
    rs2 = rs*rs
    rs3 = rs*rs2
    r2 = r*r
    r3 = r*r2
    r4 = r*r3
    r5 = r*r4
    r6 = r*r5
    r9 = r3*r6
    return sig6*A3*((sig6
                     * (+ rs3*28*(6*rs2*A2 + 15*rs*A + 10)
                        - r*rs2*945*(rs2*A2 + 2*rs*A + 1)
                        + r2*rs*1080*(2*rs2*A2 + 3*rs*A + 1)
                        - r3*420*(6*rs2*A2 + 6*rs*A + 1)
                        + r4*756*(2*rs*A2 + A)
                        - r5*378*A2)
                     - r6
                     * (+ rs3*84*(6*rs2*A2 + 15*rs*A + 10)
                        - r*rs2*3780*(rs2*A2 + 2*rs*A + 1)
                        + r2*rs*7560*(2*rs2*A2 + 3*rs*A + 1))
                     )/(252*r9)
                    - math.log(r)*10*(6*rs2*A2 + 6*rs*A + 1)
                    + r*15*(2*rs*A2 + A)
                    - r2*3*A2)


def dispersion_coefficient(sigmas, epsilons, cutoff, use_switch=False, switch_distance=0.0):
    """NonbondedForceImpl::calcDispersionCorrection (NonbondedForceImpl.cpp:236-310)."""
    n = len(sigmas)
    classes = {}
    for s, e in zip(np.asarray(sigmas).tolist(), np.asarray(epsilons).tolist()):
        classes[(s, e)] = classes.get((s, e), 0) + 1
    keys = sorted(classes)
    sum1 = sum2 = sum3 = 0.0

    def sw(sigma):
        return _eval_integral(cutoff, switch_distance, cutoff, sigma) - _eval_integral(switch_distance, switch_distance, cutoff, sigma)

    for (s, e) in keys:
        c = float(classes[(s, e)])
        c *= (c+1)/2
        s6 = s**6
        sum1 += c*e*s6*s6
        sum2 += c*e*s6
        if use_switch:
            sum3 += c*e*sw(s)
    for a in range(len(keys)):
        for b in range(a):
            s = 0.5*(keys[a][0]+keys[b][0])
            e = math.sqrt(keys[a][1]*keys[b][1])
            c = float(classes[keys[a]])*float(classes[keys[b]])
            s6 = s**6
            sum1 += c*e*s6*s6
            sum2 += c*e*s6
            if use_switch:
                sum3 += c*e*sw(s)
    ni = n*(n+1)/2.0
    sum1 /= ni
    sum2 /= ni
    sum3 /= ni
    return 8*n*n*math.pi*(sum1/(9*cutoff**9) - sum2/(3*cutoff**3) + sum3)


def _glibc_rand_stream(seed, count):
    """glibc rand() after srand(seed), via libc itself (the S1 recipe in SURVEY.md 8d uses srand(1))."""
    libc = ctypes.CDLL("libc.so.6")
    libc.srand(seed)
    rmax = 2147483647.0
    return np.array([libc.rand()/rmax for _ in range(count)])


def water_box(n=20, cutoff=0.9, method=NB_PME, jitter=0.01, rigid=True, spacing=0.3107, seed=1, ewald_tol=5e-4, name=None):
    """S1 of SURVEY.md 8(d): n^3 TIP3P waters on a cubic lattice (n=20 -> 24,000 atoms, box 6.214 nm)."""
    r_oh, theta = 0.09572, math.radians(104.52)
    nw = n**3
    N = 3*nw
    rnd = _glibc_rand_stream(seed, 3*nw) if jitter else np.zeros(3*nw)
    pos = np.zeros((N, 3))
    w = 0
    for i in range(n):
        for j in range(n):
            for k in range(n):
                c = spacing*(np.array([i, j, k]) + 0.5) + jitter*(rnd[3*w:3*w+3] - 0.5)
                pos[3*w] = c
                pos[3*w+1] = c + np.array([r_oh, 0, 0])
                pos[3*w+2] = c + np.array([r_oh*math.cos(theta), r_oh*math.sin(theta), 0])
                w += 1
    masses = np.tile([15.9994, 1.008, 1.008], nw)
    charges = np.tile([-0.834, 0.417, 0.417], nw)
    sigmas = np.tile([0.315075, 1.0, 1.0], nw)
    eps = np.tile([0.635968, 0.0, 0.0], nw)
    o = 3*np.arange(nw, dtype=np.int32)
    exc_i = np.concatenate([o, o, o+1]).astype(np.int32)
    exc_j = np.concatenate([o+1, o+2, o+2]).astype(np.int32)
    ne = len(exc_i)
    d_hh = 2*r_oh*math.sin(theta/2)
    L = n*spacing
    desc = SystemDesc(masses=masses, charges=charges, sigmas=sigmas, epsilons=eps, positions=pos,
                      box=np.diag([L, L, L]).astype(float), method=method, cutoff=cutoff, ewald_tol=ewald_tol,
                      exc_i=exc_i, exc_j=exc_j, exc_qq=np.zeros(ne), exc_sigma=np.ones(ne), exc_eps=np.zeros(ne),
                      name=name or ("water%d" % N))
    if rigid:
        desc.con_i = exc_i.copy()
        desc.con_j = exc_j.copy()
        desc.con_d = np.concatenate([np.full(nw, r_oh), np.full(nw, r_oh), np.full(nw, d_hh)])
    else:
        desc.bond_i = np.concatenate([o, o]).astype(np.int32)
        desc.bond_j = np.concatenate([o+1, o+2]).astype(np.int32)
        desc.bond_r0 = np.full(2*nw, r_oh)
        desc.bond_k = np.full(2*nw, 462750.4)
        desc.angle_i = (o+1).astype(np.int32)
        desc.angle_j = o.astype(np.int32)
        desc.angle_k = (o+2).astype(np.int32)
        desc.angle_t0 = np.full(nw, theta)
        desc.angle_kk = np.full(nw, 836.8)
    return desc


def random_ions(n=894, box=3.0, cutoff=1.0, method=NB_PME, seed=0, triclinic=False):
    """A neutral box of +-1 LJ ions on a jittered lattice (the shape of tests/nacl_amorph.dat, 894 ions, without
    reading the reference's data file); no close contacts, so forces stay in a physical range."""
    rng = np.random.default_rng(seed)
    m = int(math.ceil(n**(1.0/3.0)))
    sites = np.stack(np.meshgrid(*[np.arange(m)]*3, indexing="ij"), -1).reshape(-1, 3)
    sites = sites[rng.permutation(len(sites))[:n]]
    h = box/m
    frac = (sites + 0.5 + 0.5*(rng.random((n, 3)) - 0.5))/m
    q = np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    bx = np.diag([box, box, box]).astype(float)
    if triclinic:
        bx[1, 0] = 0.2*box
        bx[2, 0] = -0.3*box
        bx[2, 1] = 0.1*box
    pos = frac @ bx
    assert h > 0.2
    return SystemDesc(masses=np.where(q > 0, 22.99, 35.45), charges=q, sigmas=np.where(q > 0, 0.23, 0.32),
                      epsilons=np.where(q > 0, 0.0115897, 0.4184), positions=pos, box=bx, method=method, cutoff=cutoff,
                      name="ions%d" % n)


def cluster(n=70, spacing=0.32, seed=1, method=NB_NOCUTOFF, cutoff=1.0):
    """Non-periodic jittered-lattice cluster of charged LJ particles with a few exceptions (NoCutoff / CutoffNonPeriodic)."""
    rng = np.random.default_rng(seed)
    m = int(math.ceil(n**(1.0/3.0)))
    sites = np.stack(np.meshgrid(*[np.arange(m)]*3, indexing="ij"), -1).reshape(-1, 3)[:n]
    pos = (sites + 0.3*(rng.random((n, 3)) - 0.5))*spacing
    d = SystemDesc(masses=np.full(n, 10.0), charges=rng.standard_normal(n)*0.5, sigmas=np.full(n, 0.25), epsilons=rng.random(n),
                   positions=pos, box=None, method=method, cutoff=cutoff, name="cluster%d" % n)
    d.exc_i = np.array([0, 1, 5], dtype=np.int32)
    d.exc_j = np.array([1, 2, min(40, n-1)], dtype=np.int32)
    d.exc_qq = np.array([0.0, 0.1, 0.0])
    d.exc_sigma = np.array([1.0, 0.25, 1.0])
    d.exc_eps = np.array([0.0, 0.3, 0.0])
    return d


def lj_fluid(n_side=10, spacing=0.38, cutoff=1.0, method=NB_CUTOFF_PERIODIC, seed=0, charged=False):
    """Argon-like LJ lattice fluid with jitter; optionally alternating charges."""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(n_side)]*3, indexing="ij"), -1).reshape(-1, 3)
    pos = (g + 0.5)*spacing + 0.05*(rng.random(g.shape) - 0.5)
    N = len(pos)
    L = n_side*spacing
    q = np.where(np.arange(N) % 2 == 0, 0.5, -0.5) if charged else np.zeros(N)
    return SystemDesc(masses=np.full(N, 39.948), charges=q, sigmas=np.full(N, 0.34), epsilons=np.full(N, 0.997),
                      positions=pos, box=np.diag([L, L, L]).astype(float), method=method, cutoff=cutoff, name="lj%d" % N)
