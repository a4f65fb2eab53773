// bonded.cu -- harmonic bonds, harmonic angles, periodic torsions, Ryckaert-Bellemans torsions, CMAP terms, 1-4
// exceptions and the Ewald exclusion correction in ONE launch (sm_90a); custom torsions in a second launch behind it.
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

// One thread per custom torsion (CustomTorsionForce, restating ReferenceCustomTorsionIxn::calculateBondIxn): the dihedral as
// for every other torsion, dE/dtheta from the term's derivative program, the forces through torsion_force, and the energy
// program only when the energy is asked for.  A kernel of its own rather than a segment of k_bonded: the interpreter's stack
// and registers would otherwise weigh on every bonded term of every System.
__global__ void __launch_bounds__(128) k_custom_torsion(NbDev nb, CustomTorsionDev ct, int wantEnergy) {
    const int i = blockIdx.x*blockDim.x + threadIdx.x;
    double e = 0;
    if (i < ct.nslots) {
        const int p = ct.prog[i];          // uniform across the warp: the terms of one expression fill whole warps
        const unsigned char g = ct.group[i];
        if (p >= 0 && ((ct.groupMask >> (g & 31)) & 1u)) {
            const int4 at = ct.atoms[i];
            const Dihedral d = dihedral(nb, at, g & 0x80);
            const double* par = ct.params + (size_t) i*ct.paramStride;
            const double dE = custom_run(ct.code, ct.imm, ct.progStart[2*p+1], ct.progStart[2*p+2], d.theta, par, ct.globals);
            torsion_force(nb, at, d, dE);
            if (wantEnergy) e = custom_run(ct.code, ct.imm, ct.progStart[2*p], ct.progStart[2*p+1], d.theta, par, ct.globals);
        }
    }
    if (wantEnergy) {
        __shared__ double red[4];
        for (int off = 16; off > 0; off >>= 1) e += __shfl_xor_sync(0xffffffffu, e, off);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
        __syncthreads();
        if (threadIdx.x == 0) {
            const double x = red[0] + red[1] + red[2] + red[3];
            if (x != 0.0) atomicAdd(&nb.energy[EN_CUSTOM_TORSION], x);
        }
    }
}

void launch_custom_torsion(const NbDev& nb, const CustomTorsionDev& ct, bool energy, cudaStream_t s) {
    launch_high(k_custom_torsion, (ct.nslots + 127)/128, 128, 0, s, nb, ct, energy ? 1 : 0);
}

void launch_bonded(const NbDev& nb, const BondedDev& bd, const CustomTorsionDev& ct, int terms, bool energy, cudaStream_t s) {
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
    if ((terms & B200MD_TERM_CUSTOM_TORSIONS) && ct.nslots > 0) launch_custom_torsion(nb, ct, energy, s);
}
