// bonded.cu -- harmonic bonds, harmonic angles, periodic torsions, Ryckaert-Bellemans torsions, CMAP terms, 1-4
// exceptions and the Ewald exclusion correction in ONE launch (sm_90a); custom torsions, bonds, externals and angles in a
// second launch behind it, custom compound bonds in a third, custom centroid bonds in three more.
// Double precision arithmetic on fp32 positions: these terms are a few thousand work items, far below any roofline, and
// double removes them from the 1e-4 parity budget.
//
// Restates ReferenceHarmonicBondIxn / ReferenceAngleBondIxn / ReferenceProperDihedralBond / ReferenceRbDihedralBond::
// calculateBondIxn, ReferenceCMAPTorsionIxn::calculateOneIxn,
// ReferenceLJCoulomb14::calculateBondIxn (ReferenceLJCoulomb14.cpp:75-110) and the exclusion loop of
// ReferenceLJCoulombIxn::calculateEwaldIxn (ReferenceLJCoulombIxn.cpp:462-523).  Replaces the generated
// computeBondedForces kernel of CudaBondedUtilities.cpp:76-150 with pmeExclusions.cc / nonbondedExceptions.cc.
#include "engine.h"
#include "custom_interp.h"
#include "../../include/b200md.h"
#include <algorithm>

struct D3 { double x, y, z; };
__device__ __forceinline__ D3 sub(const float4& a, const float4& b) { return {(double) a.x - b.x, (double) a.y - b.y, (double) a.z - b.z}; }
__device__ __forceinline__ D3 cross(const D3& a, const D3& b) { return {a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x}; }
__device__ __forceinline__ double dot(const D3& a, const D3& b) { return a.x*b.x + a.y*b.y + a.z*b.z; }
__device__ __forceinline__ D3 scale(const D3& a, double s) { return {a.x*s, a.y*s, a.z*s}; }

__device__ __forceinline__ void add_force(const NbDev& nb, int a, const D3& f) {
    atomicAdd((unsigned long long*) &nb.force[a], (unsigned long long) __double2ll_rn(f.x*B200MD_FORCE_SCALE));
    atomicAdd((unsigned long long*) &nb.force[a + nb.npad], (unsigned long long) __double2ll_rn(f.y*B200MD_FORCE_SCALE));
    atomicAdd((unsigned long long*) &nb.force[a + 2*nb.npad], (unsigned long long) __double2ll_rn(f.z*B200MD_FORCE_SCALE));
}

__device__ __forceinline__ D3 min_image_d(D3 d, const BoxDev& b) {
    double s = floor(d.z*(double) b.invCz + 0.5);
    d.x -= s*b.cx; d.y -= s*b.cy; d.z -= s*b.cz;
    s = floor(d.y*(double) b.invBy + 0.5);
    d.x -= s*b.bx; d.y -= s*b.by;
    s = floor(d.x*(double) b.invAx + 0.5);
    d.x -= s*b.ax;
    return d;
}

// Dihedral of the atoms (x, y, z, w) (ReferenceBondIxn::getDihedralAngleBetweenThreeVectors): the three difference vectors,
// the two plane normals and their squared norms, the clamped cosine of the angle and the signed angle in (-pi, pi].
struct Dihedral { D3 v0, v1, v2, cp0, cp1; double n0, n1, c, theta; };
__device__ __forceinline__ Dihedral dihedral(const NbDev& nb, const int4& at, bool periodic) {
    Dihedral d;
    d.v0 = sub(nb.posq[at.x], nb.posq[at.y]);
    d.v1 = sub(nb.posq[at.z], nb.posq[at.y]);
    d.v2 = sub(nb.posq[at.z], nb.posq[at.w]);
    if (periodic) { d.v0 = min_image_d(d.v0, nb.box); d.v1 = min_image_d(d.v1, nb.box); d.v2 = min_image_d(d.v2, nb.box); }
    d.cp0 = cross(d.v0, d.v1); d.cp1 = cross(d.v1, d.v2);
    d.n0 = dot(d.cp0, d.cp0); d.n1 = dot(d.cp1, d.cp1);
    double c = dot(d.cp0, d.cp1)/sqrt(d.n0*d.n1);
    c = fmin(1.0, fmax(-1.0, c));
    double theta;
    if (c > 0.99 || c < -0.99) {
        // near 0 / pi use the cross product for accuracy (ReferenceBondIxn::getAngleBetweenTwoVectors)
        D3 cc = cross(d.cp0, d.cp1);
        double sc = sqrt(dot(cc, cc)/(d.n0*d.n1));
        theta = asin(fmin(1.0, sc));
        if (c < 0) theta = 3.14159265358979323846 - theta;
    }
    else theta = acos(c);
    if (dot(d.v0, d.cp1) < 0) theta = -theta;
    d.c = c; d.theta = theta;
    return d;
}

// Forces of an energy term of one dihedral with derivative dE = dE/dtheta, distributed over its four atoms as in
// ReferenceProperDihedralBond::calculateBondIxn.
__device__ __forceinline__ void torsion_force(const NbDev& nb, const int4& at, const Dihedral& d, double dE) {
    const double nbc2 = dot(d.v1, d.v1), nbc = sqrt(nbc2);
    const double ffx = -dE*nbc/d.n0, ffw = dE*nbc/d.n1;
    const double ffy = dot(d.v0, d.v1)/nbc2, ffz = dot(d.v2, d.v1)/nbc2;
    D3 f1 = scale(d.cp0, ffx), f4 = scale(d.cp1, ffw);
    D3 s = {ffy*f1.x - ffz*f4.x, ffy*f1.y - ffz*f4.y, ffy*f1.z - ffz*f4.z};
    add_force(nb, at.x, f1);
    add_force(nb, at.y, {s.x-f1.x, s.y-f1.y, s.z-f1.z});
    add_force(nb, at.z, {-s.x-f4.x, -s.y-f4.y, -s.z-f4.z});
    add_force(nb, at.w, f4);
}

__global__ void __launch_bounds__(128) k_bonded(NbDev nb, BondedDev bd, int terms, int wantEnergy) {
    const int nB = (terms & B200MD_TERM_BONDS) ? bd.nbonds : 0;
    const int nA = (terms & B200MD_TERM_ANGLES) ? bd.nangles : 0;
    const int nT = (terms & B200MD_TERM_TORSIONS) ? bd.ntorsions : 0;
    const int nR = (terms & B200MD_TERM_RB_TORSIONS) ? bd.nrb : 0;
    const int nC = (terms & B200MD_TERM_CMAP) ? bd.ncmap : 0;
    // both the 1-4 pairs and the Ewald exclusion correction belong to the DIRECT-space group: the reference evaluates
    // the exclusion loop after `if (!includeDirect) return;` (ReferenceLJCoulombIxn.cpp:373-374, 462-523)
    const bool doDirect = (terms & B200MD_TERM_NB_DIRECT) != 0;
    const bool doRecip = doDirect && nb.method == B200MD_NB_PME;
    const int nE = doDirect ? bd.nexc : 0;
    // the bonded work is sharded over ranks in the multi-GPU force decomposition
    const int gid = nb.rank + nb.world*(blockIdx.x*blockDim.x + threadIdx.x);
    double eB = 0, eA = 0, eT = 0, eR = 0, eC = 0, eE = 0;
    int i = gid;
    // group byte of a bonded term: bits 0-4 force group, bit 7 = the Force uses periodic boundary conditions
    // (usesPeriodicBoundaryConditions: every difference vector takes the minimum image, ReferenceBondIxn / getDeltaRPeriodic)
    if (i < nB && ((bd.groupMask >> (bd.bondGroup[i] & 31)) & 1u)) {
        const int2 at = bd.bondAtoms[i];
        const double2 pr = bd.bondParams[i];
        D3 d = sub(nb.posq[at.x], nb.posq[at.y]);
        if (bd.bondGroup[i] & 0x80) d = min_image_d(d, nb.box);
        const double r = sqrt(dot(d, d));
        const double dr = r - pr.x;
        eB = 0.5*pr.y*dr*dr;
        const double s = (r > 0) ? -pr.y*dr/r : 0.0;
        add_force(nb, at.x, scale(d, s));
        add_force(nb, at.y, scale(d, -s));
    }
    i -= nB;
    if (i >= 0 && i < nA && ((bd.groupMask >> (bd.angleGroup[i] & 31)) & 1u)) {
        const int4 at = bd.angleAtoms[i];
        const double2 pr = bd.angleParams[i];
        D3 v0 = sub(nb.posq[at.y], nb.posq[at.x]);
        D3 v1 = sub(nb.posq[at.y], nb.posq[at.z]);
        if (bd.angleGroup[i] & 0x80) { v0 = min_image_d(v0, nb.box); v1 = min_image_d(v1, nb.box); }
        D3 cp = cross(v0, v1);
        double rp = sqrt(dot(cp, cp));
        rp = fmax(rp, 1e-6);
        const double r21 = dot(v0, v0), r23 = dot(v1, v1);
        double c = dot(v0, v1)/sqrt(r21*r23);
        c = fmin(1.0, fmax(-1.0, c));
        const double theta = acos(c);
        const double dth = theta - pr.x;
        eA = 0.5*pr.y*dth*dth;
        const double dE = pr.y*dth;
        D3 f1 = scale(cross(v0, cp), dE/(r21*rp));
        D3 f3 = scale(cross(cp, v1), dE/(r23*rp));
        add_force(nb, at.x, f1);
        add_force(nb, at.z, f3);
        add_force(nb, at.y, {-f1.x-f3.x, -f1.y-f3.y, -f1.z-f3.z});
    }
    i -= nA;
    if (i >= 0 && i < nT && ((bd.groupMask >> (bd.torsionGroup[i] & 31)) & 1u)) {
        const int4 at = bd.torsionAtoms[i];
        const double4 pr = bd.torsionParams[i];   // k, phase, n
        const Dihedral d = dihedral(nb, at, bd.torsionGroup[i] & 0x80);
        const double arg = pr.z*d.theta - pr.y;
        eT = pr.x*(1.0 + cos(arg));
        torsion_force(nb, at, d, -pr.x*pr.z*sin(arg));
    }
    i -= nT;
    if (i >= 0 && i < nR && ((bd.groupMask >> (bd.rbGroup[i] & 31)) & 1u)) {
        // ReferenceRbDihedralBond::calculateBondIxn: polymer convention psi = phi - pi, E = sum_n c_n cos^n psi
        const int4 at = bd.rbAtoms[i];
        const double* cn = bd.rbParams + 6*i;
        const Dihedral d = dihedral(nb, at, bd.rbGroup[i] & 0x80);
        const double psi = d.theta < 0 ? d.theta + 3.14159265358979323846 : d.theta - 3.14159265358979323846;
        const double cpsi = -d.c;
        double dE = 0, e = cn[0], cf = 1.0;
        for (int n = 1; n < 6; n++) {
            dE -= n*cn[n]*cf;
            cf *= cpsi;
            e += cf*cn[n];
        }
        eR = e;
        torsion_force(nb, at, d, dE*sin(psi));
    }
    i -= nR;
    if (i >= 0 && i < nC && ((bd.groupMask >> (bd.cmapGroup[i] & 31)) & 1u)) {
        // ReferenceCMAPTorsionIxn::calculateOneIxn: bicubic patch of the map at the two dihedrals, each taken in [0, 2 pi)
        const int4 atA = bd.cmapAtoms[2*i], atB = bd.cmapAtoms[2*i+1];
        const bool periodic = bd.cmapGroup[i] & 0x80;
        // the second dihedral is evaluated again for its forces rather than kept across the spline: fewer live registers
        const Dihedral dA = dihedral(nb, atA, periodic);
        const double twoPi = 2.0*3.14159265358979323846;
        const double angleA = fmod(dA.theta + twoPi, twoPi), angleB = fmod(dihedral(nb, atB, periodic).theta + twoPi, twoPi);
        const int2 map = bd.cmapMaps[bd.cmapMap[i]];      // (first patch, size)
        const double delta = twoPi/map.y;
        const int s = (int) fmin(angleA/delta, (double) (map.y - 1));
        const int t = (int) fmin(angleB/delta, (double) (map.y - 1));
        const double* c = bd.cmapCoeff + 16*((size_t) map.x + s + map.y*t);
        const double da = angleA/delta - s, db = angleB/delta - t;
        double e = 0, dEdA = 0, dEdB = 0;
        for (int k = 3; k >= 0; k--) {
            e = da*e + ((c[k*4+3]*db + c[k*4+2])*db + c[k*4+1])*db + c[k*4+0];
            dEdA = db*dEdA + (3.0*c[k+3*4]*da + 2.0*c[k+2*4])*da + c[k+1*4];
            dEdB = da*dEdB + (3.0*c[k*4+3]*db + 2.0*c[k*4+2])*db + c[k*4+1];
        }
        eC = e;
        torsion_force(nb, atA, dA, dEdA/delta);
        torsion_force(nb, atB, dihedral(nb, atB, periodic), dEdB/delta);
    }
    i -= nC;
    if (i >= 0 && i < nE) {
        const int2 at = bd.excAtoms[i];
        const double4 pr = bd.excParams[i];       // (k qq14, sigma, 4 eps, k qi qj)
        D3 d = sub(nb.posq[at.x], nb.posq[at.y]); // x_i - x_j
        if (bd.excPeriodic && nb.box.periodic) d = min_image_d(d, nb.box);
        const double r2 = dot(d, d);
        const double invR = 1.0/sqrt(r2);
        double dEdR = 0, e = 0;
        if (doDirect && (pr.x != 0.0 || pr.z != 0.0)) {
            // ReferenceLJCoulomb14::calculateBondIxn
            double s2 = pr.y*invR; s2 *= s2;
            const double s6 = s2*s2*s2;
            dEdR += (pr.z*(12.0*s6 - 6.0)*s6 + pr.x*invR)*invR*invR;
            e += pr.z*(s6 - 1.0)*s6 + pr.x*invR;
        }
        if (doRecip && pr.w != 0.0) {
            const double r = r2*invR;
            const double ar = (double) nb.alpha*r;
            const double er = erf(ar);
            if (er > 1e-6) {
                dEdR -= pr.w*invR*invR*invR*(er - 1.12837916709551257390*ar*exp(-ar*ar));
                e -= pr.w*invR*er;
            }
            else
                e -= (double) nb.alpha*1.12837916709551257390*pr.w;
        }
        eE = e;
        add_force(nb, at.x, scale(d, dEdR));
        add_force(nb, at.y, scale(d, -dEdR));
    }
    if (wantEnergy) {
        // block reduction of the six partial energies
        __shared__ double red[6][4];
        double v[6] = {eB, eA, eT, eE, eR, eC};
        for (int k = 0; k < 6; k++) {
            double x = v[k];
            for (int off = 16; off > 0; off >>= 1) x += __shfl_xor_sync(0xffffffffu, x, off);
            if ((threadIdx.x & 31) == 0) red[k][threadIdx.x >> 5] = x;
        }
        __syncthreads();
        if (threadIdx.x < 6) {
            double x = red[threadIdx.x][0] + red[threadIdx.x][1] + red[threadIdx.x][2] + red[threadIdx.x][3];
            const int slot[6] = {EN_BOND, EN_ANGLE, EN_TORSION, EN_EXC, EN_RBTORSION, EN_CMAP};
            if (x != 0.0) atomicAdd(&nb.energy[slot[threadIdx.x]], x);
        }
    }
}

// One thread per custom term (restating ReferenceCustomTorsionIxn / ReferenceCustomBondIxn / ReferenceCustomAngleIxn::
// calculateBondIxn and ReferenceCustomExternalIxn::calculateForce).  A torsion: the dihedral as for every other torsion, dE/dtheta from the term's
// derivative program, the forces through torsion_force.  A bond: r = |x_b - x_a|, dE/dr, (dE/dr)/r (x_b - x_a) on a and its
// negative on b.  An angle: the angle and its forces as the harmonic-angle segment of k_bonded computes them, with dE/dtheta
// from the derivative program.  An external: the particle's continuous coordinate (posq plus cellOffset lattice vectors, what
// b200md_get_positions reports: the molecule wrap of the list build must not move a restraint), minus the three derivatives.
// The energy program runs only when the energy is asked for, and a class only when its bit is in `terms`.  A kernel of its
// own rather than a segment of k_bonded: the interpreter's stack and registers would otherwise weigh on every bonded term of
// every System.
__global__ void __launch_bounds__(128) k_custom(NbDev nb, CustomDev ct, int terms, int wantEnergy) {
    const int i = blockIdx.x*blockDim.x + threadIdx.x;
    double e = 0;
    if (i < ct.nslots) {
        const int p = ct.expr[i];          // uniform across the warp: the terms of one expression fill whole warps
        const unsigned char g = ct.group[i];
        const int cls = p >= 0 ? ct.exprClass[p] : 0;
        const int bit = cls == B200MD_CUSTOM_TORSION ? B200MD_TERM_CUSTOM_TORSIONS :
                        cls == B200MD_CUSTOM_BOND ? B200MD_TERM_CUSTOM_BONDS :
                        cls == B200MD_CUSTOM_ANGLE ? B200MD_TERM_CUSTOM_ANGLES : B200MD_TERM_CUSTOM_EXTERNALS;
        if (p >= 0 && (terms & bit) && ((ct.groupMask >> (g & 31)) & 1u)) {
            const int4 at = ct.atoms[i];
            const double* par = ct.params + (size_t) i*ct.paramStride;
            const int q = ct.exprProg[p];
            // periodicdistance reduces by the box the pair terms use (a barostat's box reaches it the same way)
            const CustomBox box = {nb.box.dax, nb.box.bx, nb.box.dby, nb.box.cx, nb.box.cy, nb.box.dcz};
            double v[3];
            if (cls == B200MD_CUSTOM_TORSION) {
                const Dihedral d = dihedral(nb, at, g & 0x80);
                v[0] = d.theta;
                const double dE = custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q+1], ct.progStart[q+2], v, par, ct.globals, box);
                torsion_force(nb, at, d, dE);
            }
            else if (cls == B200MD_CUSTOM_BOND) {
                D3 d = sub(nb.posq[at.y], nb.posq[at.x]);
                if (g & 0x80) d = min_image_d(d, nb.box);
                v[0] = sqrt(dot(d, d));
                const double dE = custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q+1], ct.progStart[q+2], v, par, ct.globals, box);
                const double s = v[0] > 0 ? dE/v[0] : 0.0;
                add_force(nb, at.x, scale(d, s));
                add_force(nb, at.y, scale(d, -s));
            }
            else if (cls == B200MD_CUSTOM_ANGLE) {
                D3 v0 = sub(nb.posq[at.y], nb.posq[at.x]);
                D3 v1 = sub(nb.posq[at.y], nb.posq[at.z]);
                if (g & 0x80) { v0 = min_image_d(v0, nb.box); v1 = min_image_d(v1, nb.box); }
                D3 cp = cross(v0, v1);
                double rp = sqrt(dot(cp, cp));
                rp = fmax(rp, 1e-6);
                const double r21 = dot(v0, v0), r23 = dot(v1, v1);
                double c = dot(v0, v1)/sqrt(r21*r23);
                c = fmin(1.0, fmax(-1.0, c));
                v[0] = acos(c);
                const double dE = custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q+1], ct.progStart[q+2], v, par, ct.globals, box);
                D3 f1 = scale(cross(v0, cp), dE/(r21*rp));
                D3 f3 = scale(cross(cp, v1), dE/(r23*rp));
                add_force(nb, at.x, f1);
                add_force(nb, at.z, f3);
                add_force(nb, at.y, {-f1.x-f3.x, -f1.y-f3.y, -f1.z-f3.z});
            }
            else {
                const float4 x = nb.posq[at.x];
                v[0] = x.x; v[1] = x.y; v[2] = x.z;
                const int kx = nb.cellOffset[at.x], ky = nb.cellOffset[at.x + nb.npad], kz = nb.cellOffset[at.x + 2*nb.npad];
                v[0] += kx*nb.box.dax + ky*(double) nb.box.bx + kz*(double) nb.box.cx;
                v[1] += ky*nb.box.dby + kz*(double) nb.box.cy;
                v[2] += kz*nb.box.dcz;
                D3 f;
                f.x = -custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q+1], ct.progStart[q+2], v, par, ct.globals, box);
                f.y = -custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q+2], ct.progStart[q+3], v, par, ct.globals, box);
                f.z = -custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q+3], ct.progStart[q+4], v, par, ct.globals, box);
                add_force(nb, at.x, f);
            }
            if (wantEnergy) e = custom_run<B200MD_CUSTOM_MAX_STACK, false>(ct.code, ct.imm, ct.progStart[q], ct.progStart[q+1], v, par, ct.globals, box);
        }
    }
    if (wantEnergy) {
        __shared__ double red[4];
        for (int off = 16; off > 0; off >>= 1) e += __shfl_xor_sync(0xffffffffu, e, off);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
        __syncthreads();
        if (threadIdx.x == 0) {
            const double x = red[0] + red[1] + red[2] + red[3];
            if (x != 0.0) atomicAdd(&nb.energy[EN_CUSTOM], x);
        }
    }
}

void launch_custom(const NbDev& nb, const CustomDev& ct, int terms, bool energy, cudaStream_t s) {
    launch_high(k_custom, (ct.nslots + 127)/128, 128, 0, s, nb, ct, terms, energy ? 1 : 0);
}

// Where k_compound's particles come from and where a derivative program's value goes.  CompoundAtoms: a particle is an
// atom, read at its continuous coordinate (posq plus cellOffset lattice vectors, what b200md_get_positions reports), and minus
// the derivative is added to its force at once.  CentroidCenters: a particle is a group centre of k_centroid_centers, and
// derivative j of slot i is stored to deriv[i][j-1] for k_centroid_scatter, every one of them in every evaluation (a CONST 0
// program stores 0), so that the scatter never reads a value of an earlier evaluation.
struct CompoundAtoms {
    static constexpr bool STORE_ALL = false;
    __device__ __forceinline__ void coords(const NbDev& nb, int a, double* v) const {
        const float4 x = nb.posq[a];
        const int kx = nb.cellOffset[a], ky = nb.cellOffset[a + nb.npad], kz = nb.cellOffset[a + 2*nb.npad];
        v[0] = x.x + (kx*nb.box.dax + ky*(double) nb.box.bx + kz*(double) nb.box.cx);
        v[1] = x.y + (ky*nb.box.dby + kz*(double) nb.box.cy);
        v[2] = x.z + kz*nb.box.dcz;
    }
    __device__ __forceinline__ void store(const NbDev& nb, const int* at, int i, int j, double r) const {
        atomicAdd((unsigned long long*) &nb.force[at[(j-1)/3] + ((j-1) % 3)*nb.npad], (unsigned long long) __double2ll_rn(-r*B200MD_FORCE_SCALE));
    }
};
struct CentroidCenters {
    static constexpr bool STORE_ALL = true;
    const double* center; double* deriv;
    __device__ __forceinline__ void coords(const NbDev&, int g, double* v) const {
        v[0] = center[3*g]; v[1] = center[3*g+1]; v[2] = center[3*g+2];
    }
    __device__ __forceinline__ void store(const NbDev&, const int*, int i, int j, double r) const {
        deriv[(size_t) i*CENTROID_DERIVS + j - 1] = r;
    }
};

// Custom compound bonds (restating ReferenceCustomCompoundBondIxn::calculateOneIxn): the energy is a function of the 3 N
// coordinates of the term's N particles, the force on particle k minus the derivatives by its three.  One thread per (term,
// program): warp W runs program W % COMPOUND_PROGRAMS (0 the energy, 1 + 3 k + c the derivative by coordinate c of particle
// k) for the 32 slots of group W / COMPOUND_PROGRAMS, so a warp still runs one program with uniform code loads, and the
// programs of a term, which do not depend on each other, run side by side: a lone six-particle restraint takes the time of
// its longest program, not of all 19.  The coordinates are the continuous ones (posq plus cellOffset lattice vectors, what
// b200md_get_positions reports): an expression may read them directly, and a non-periodic restraint between two molecules
// must not jump when the list build wraps one of them.  A derivative program that is the single instruction CONST 0 is not
// run and adds nothing.  A kernel of its own: its interpreter holds a 32-deep stack and the three point functions, which
// k_custom's terms never need.  Src (CompoundAtoms, CentroidCenters above) says what a particle is: custom centroid bonds
// run the same programs at group centres.
#define COMPOUND_PROGRAMS (1 + 3*B200MD_CUSTOM_MAX_PARTICLES)
template <class Src>
__global__ void __launch_bounds__(128) k_compound(NbDev nb, CompoundDev cd, int wantEnergy, Src src) {
    const int warp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
    const int j = warp % COMPOUND_PROGRAMS, i = (warp/COMPOUND_PROGRAMS)*32 + (threadIdx.x & 31);
    double e = 0;
    if (i < cd.nslots && (j > 0 || wantEnergy)) {
        const int p = cd.expr[i];          // uniform across the warp: the terms of one expression fill whole warps
        if (p >= 0 && j <= 3*cd.exprParticles[p] && ((cd.groupMask >> (cd.group[i] & 31)) & 1u)) {
            const int np = cd.exprParticles[p], q = cd.exprProg[p] + j;
            const int begin = cd.progStart[q], end = cd.progStart[q+1];
            if (j == 0 || !(end - begin == 1 && cd.code[begin].x == B200MD_OP_CONST && cd.imm[begin] == 0.0)) {
                const int* at = cd.atoms + B200MD_CUSTOM_MAX_PARTICLES*(size_t) i;
                const CustomBox box = {nb.box.dax, nb.box.bx, nb.box.dby, nb.box.cx, nb.box.cy, nb.box.dcz};
                double v[3*B200MD_CUSTOM_MAX_PARTICLES];
                for (int k = 0; k < np; k++) src.coords(nb, at[k], v + 3*k);
                const double r = custom_run<B200MD_CUSTOM_COMPOUND_MAX_STACK, true>(cd.code, cd.imm, begin, end, v, cd.params + (size_t) i*cd.paramStride,
                                                                                    cd.globals, box, cd.exprPeriodic[p] != 0);
                if (j == 0) e = r;
                else src.store(nb, at, i, j, r);
            }
            else if (Src::STORE_ALL) src.store(nb, nullptr, i, j, 0.0);
        }
    }
    if (wantEnergy) {
        __shared__ double red[4];
        for (int off = 16; off > 0; off >>= 1) e += __shfl_xor_sync(0xffffffffu, e, off);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
        __syncthreads();
        if (threadIdx.x == 0) {
            const double x = red[0] + red[1] + red[2] + red[3];
            if (x != 0.0) atomicAdd(&nb.energy[EN_CUSTOM], x);
        }
    }
}

void launch_compound(const NbDev& nb, const CompoundDev& cd, bool energy, cudaStream_t s) {
    const int warps = cd.nslots/32*COMPOUND_PROGRAMS;      // nslots is a whole number of warps
    launch_high(k_compound<CompoundAtoms>, (warps + 3)/4, 128, 0, s, nb, cd, energy ? 1 : 0, CompoundAtoms{});
}

// Custom centroid bonds (restating ReferenceCustomCentroidBondIxn::calculateIxn), in three kernels.  k_centroid_centers:
// one warp per group, its lanes striding over the group's atoms, each summing w x of their continuous coordinates (those of
// CompoundAtoms, so that a single-atom group of weight 1 is exactly its atom's coordinate), then a fixed xor-shuffle tree:
// the centres do not depend on timing, bit for bit.  The programs: k_compound<CentroidCenters>.  k_centroid_scatter: one
// thread per scatter entry (slot, position k of the group in the bond, atom, weight w; in slot order, weight-0 entries dropped
// on the host), adding -w times the three derivatives by the centre of group k to the atom's force through the fixed-point
// atomics, whose integer sums do not depend on their order.
__global__ void __launch_bounds__(128) k_centroid_centers(NbDev nb, CentroidDev cn) {
    const int g = (blockIdx.x*blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (g >= cn.ngroups) return;           // whole warps
    double c[3] = {0.0, 0.0, 0.0};
    for (int k = cn.groupStart[g] + lane; k < cn.groupStart[g+1]; k += 32) {
        double x[3];
        CompoundAtoms().coords(nb, cn.groupAtoms[k], x);
        const double w = cn.groupWeight[k];
        c[0] += w*x[0]; c[1] += w*x[1]; c[2] += w*x[2];
    }
    for (int off = 16; off > 0; off >>= 1)
        for (int d = 0; d < 3; d++) c[d] += __shfl_xor_sync(0xffffffffu, c[d], off);
    if (lane == 0) { cn.center[3*g] = c[0]; cn.center[3*g+1] = c[1]; cn.center[3*g+2] = c[2]; }
}

__global__ void __launch_bounds__(128) k_centroid_scatter(NbDev nb, CompoundDev cd, CentroidDev cn) {
    const int t = blockIdx.x*blockDim.x + threadIdx.x;
    if (t >= cn.nscatter) return;
    const int4 s = cn.scatter[t];          // (slot, group position k, atom, 0)
    if (!((cd.groupMask >> (cd.group[s.x] & 31)) & 1u)) return;
    const double w = cn.scatterWeight[t];
    const double* d = cn.deriv + (size_t) s.x*CENTROID_DERIVS + 3*s.y;
    for (int c = 0; c < 3; c++)
        atomicAdd((unsigned long long*) &nb.force[s.z + c*nb.npad], (unsigned long long) __double2ll_rn(-(w*d[c])*B200MD_FORCE_SCALE));
}

void launch_centroid(const NbDev& nb, const CompoundDev& cd, const CentroidDev& cn, bool energy, cudaStream_t s) {
    launch_high(k_centroid_centers, (cn.ngroups + 3)/4, 128, 0, s, nb, cn);
    const int warps = cd.nslots/32*COMPOUND_PROGRAMS;
    launch_high(k_compound<CentroidCenters>, (warps + 3)/4, 128, 0, s, nb, cd, energy ? 1 : 0, CentroidCenters{cn.center, cn.deriv});
    launch_high(k_centroid_scatter, std::max(1, (cn.nscatter + 127)/128), 128, 0, s, nb, cd, cn);
}

void launch_bonded(const NbDev& nb, const BondedDev& bd, const CustomDev& ct, const CompoundDev& cd, const CompoundDev& cc, const CentroidDev& cn,
                   int terms, bool energy, cudaStream_t s) {
    int n = 0;
    if (terms & B200MD_TERM_BONDS) n += bd.nbonds;
    if (terms & B200MD_TERM_ANGLES) n += bd.nangles;
    if (terms & B200MD_TERM_TORSIONS) n += bd.ntorsions;
    if (terms & B200MD_TERM_RB_TORSIONS) n += bd.nrb;
    if (terms & B200MD_TERM_CMAP) n += bd.ncmap;
    if (terms & B200MD_TERM_NB_DIRECT) n += bd.nexc;
    if (n > 0) {
        int per = (n + nb.world - 1)/nb.world;
        launch_high(k_bonded, (per + 127)/128, 128, 0, s, nb, bd, terms, energy ? 1 : 0);
    }
    if (terms & ct.terms) launch_custom(nb, ct, terms, energy, s);
    if ((terms & B200MD_TERM_CUSTOM_COMPOUND) && cd.nslots > 0) launch_compound(nb, cd, energy, s);
    if ((terms & B200MD_TERM_CUSTOM_CENTROID) && cc.nslots > 0) launch_centroid(nb, cc, cn, energy, s);
}
