// integrate.cu -- fused integrate + constrain step (sm_90a): one lane per atom, 4 lanes per integration unit
// (a rigid 3-atom molecule, an X-H_n SHAKE cluster or a free atom), everything in registers, ONE launch.
//
// Restates ReferenceStochasticDynamics::update (ReferenceStochasticDynamics.cpp:89-194),
// ReferenceLangevinMiddleDynamics::update (ReferenceLangevinMiddleDynamics.cpp:54-127), ReferenceVerletDynamics,
// ReferenceSETTLEAlgorithm::apply/applyToVelocities (ReferenceSETTLEAlgorithm.cpp:54-244) and the per-cluster SHAKE of
// the reference GPU platforms (integrationUtilities.cc:99-326).  Replaces integrateLangevinPart1 -> applySettle* ->
// applyShake* -> integrateLangevinPart2 -> generateRandomNumbers (4-6 launches + an RNG refill) with one kernel;
// the noise is Philox4x32-10 keyed on (seed; atom, step) so results do not depend on launch geometry.
//
// Every kernel here is templated on the working type R: float in a single-precision context, double in a mixed-precision
// one (positions hi + lo, velocities and constraint constants in double; engine.h "integration state").  The float
// instantiations are the same arithmetic as before the template existed.
#include "engine.h"
#include <algorithm>
#include "../../include/b200md.h"

template <class R> struct V3 { R x, y, z; };
template <class R> __device__ __forceinline__ V3<R> operator+(V3<R> a, V3<R> b) { return {a.x+b.x, a.y+b.y, a.z+b.z}; }
template <class R> __device__ __forceinline__ V3<R> operator-(V3<R> a, V3<R> b) { return {a.x-b.x, a.y-b.y, a.z-b.z}; }
template <class R> __device__ __forceinline__ V3<R> operator*(V3<R> a, R s) { return {a.x*s, a.y*s, a.z*s}; }
template <class R> __device__ __forceinline__ R dot(V3<R> a, V3<R> b) { return a.x*b.x + a.y*b.y + a.z*b.z; }

// ---------------------------------------------------------------- SETTLE, positions (Miyamoto & Kollman 1992)
// NOTE on provenance: settle_positions / settle_velocities below restate the published closed form in the same sequence of
// steps (and with the same intermediate names) as the reference's GPU kernels applySettleToPositions / applySettleToVelocities
// (platforms/common/src/kernels/integrationUtilities.cc:328-470, 489-551), which themselves follow
// ReferenceSETTLEAlgorithm.cpp:54-244; only the types (registers of the working type, one thread per water inside the fused
// integrate kernel) and the surrounding kernel are this repository's own.  The SHAKE code further down is restructured
// (looped, per-constraint distances).
// x: old positions (constraints satisfied), d: position deltas (in/out), m: masses, dist1 = |01| = |02|, dist2 = |12|
template <class R>
__device__ void settle_positions(const V3<R>* x, V3<R>* d, const R* m, R dist1, R dist2) {
    const V3<R> xp0 = d[0], xp1 = d[1], xp2 = d[2];
    const R xb0 = x[1].x-x[0].x, yb0 = x[1].y-x[0].y, zb0 = x[1].z-x[0].z;
    const R xc0 = x[2].x-x[0].x, yc0 = x[2].y-x[0].y, zc0 = x[2].z-x[0].z;
    const R invTotalMass = R(1)/(m[0]+m[1]+m[2]);
    const R xcom = (xp0.x*m[0] + (xb0+xp1.x)*m[1] + (xc0+xp2.x)*m[2])*invTotalMass;
    const R ycom = (xp0.y*m[0] + (yb0+xp1.y)*m[1] + (yc0+xp2.y)*m[2])*invTotalMass;
    const R zcom = (xp0.z*m[0] + (zb0+xp1.z)*m[1] + (zc0+xp2.z)*m[2])*invTotalMass;
    const R xa1 = xp0.x - xcom, ya1 = xp0.y - ycom, za1 = xp0.z - zcom;
    const R xb1 = xb0 + xp1.x - xcom, yb1 = yb0 + xp1.y - ycom, zb1 = zb0 + xp1.z - zcom;
    const R xc1 = xc0 + xp2.x - xcom, yc1 = yc0 + xp2.y - ycom, zc1 = zc0 + xp2.z - zcom;
    const R xaksZd = yb0*zc0 - zb0*yc0, yaksZd = zb0*xc0 - xb0*zc0, zaksZd = xb0*yc0 - yb0*xc0;
    const R xaksXd = ya1*zaksZd - za1*yaksZd, yaksXd = za1*xaksZd - xa1*zaksZd, zaksXd = xa1*yaksZd - ya1*xaksZd;
    const R xaksYd = yaksZd*zaksXd - zaksZd*yaksXd, yaksYd = zaksZd*xaksXd - xaksZd*zaksXd, zaksYd = xaksZd*yaksXd - yaksZd*xaksXd;
    const R axlng = rsqrt_r(xaksXd*xaksXd + yaksXd*yaksXd + zaksXd*zaksXd);
    const R aylng = rsqrt_r(xaksYd*xaksYd + yaksYd*yaksYd + zaksYd*zaksYd);
    const R azlng = rsqrt_r(xaksZd*xaksZd + yaksZd*yaksZd + zaksZd*zaksZd);
    const R t11 = xaksXd*axlng, t21 = yaksXd*axlng, t31 = zaksXd*axlng;
    const R t12 = xaksYd*aylng, t22 = yaksYd*aylng, t32 = zaksYd*aylng;
    const R t13 = xaksZd*azlng, t23 = yaksZd*azlng, t33 = zaksZd*azlng;
    const R xb0d = t11*xb0 + t21*yb0 + t31*zb0, yb0d = t12*xb0 + t22*yb0 + t32*zb0;
    const R xc0d = t11*xc0 + t21*yc0 + t31*zc0, yc0d = t12*xc0 + t22*yc0 + t32*zc0;
    const R za1d = t13*xa1 + t23*ya1 + t33*za1;
    const R xb1d = t11*xb1 + t21*yb1 + t31*zb1, yb1d = t12*xb1 + t22*yb1 + t32*zb1, zb1d = t13*xb1 + t23*yb1 + t33*zb1;
    const R xc1d = t11*xc1 + t21*yc1 + t31*zc1, yc1d = t12*xc1 + t22*yc1 + t32*zc1, zc1d = t13*xc1 + t23*yc1 + t33*zc1;
    // step 2
    const R rc = R(0.5)*dist2;
    R rb = sqrt_r(dist1*dist1 - rc*rc);
    const R ra = rb*(m[1]+m[2])*invTotalMass;
    rb -= ra;
    const R sinphi = za1d/ra;
    const R cosphi = sqrt_r(R(1) - sinphi*sinphi);
    const R sinpsi = (zb1d - zc1d)/(R(2)*rc*cosphi);
    const R cospsi = sqrt_r(R(1) - sinpsi*sinpsi);
    const R ya2d = ra*cosphi;
    R xb2d = -rc*cospsi;
    const R yb2d = -rb*cosphi - rc*sinpsi*sinphi;
    const R yc2d = -rb*cosphi + rc*sinpsi*sinphi;
    const R xb2d2 = xb2d*xb2d;
    const R hh2 = R(4)*xb2d2 + (yb2d-yc2d)*(yb2d-yc2d) + (zb1d-zc1d)*(zb1d-zc1d);
    const R deltx = R(2)*xb2d + sqrt_r(R(4)*xb2d2 - hh2 + dist2*dist2);
    xb2d -= deltx*R(0.5);
    // step 3
    const R alpha = xb2d*(xb0d-xc0d) + yb0d*yb2d + yc0d*yc2d;
    const R beta = xb2d*(yc0d-yb0d) + xb0d*yb2d + xc0d*yc2d;
    const R gamma = xb0d*yb1d - xb1d*yb0d + xc0d*yc1d - xc1d*yc0d;
    const R al2be2 = alpha*alpha + beta*beta;
    const R sintheta = (alpha*gamma - beta*sqrt_r(al2be2 - gamma*gamma))/al2be2;
    // step 4
    const R costheta = sqrt_r(R(1) - sintheta*sintheta);
    const R xa3d = -ya2d*sintheta, ya3d = ya2d*costheta, za3d = za1d;
    const R xb3d = xb2d*costheta - yb2d*sintheta, yb3d = xb2d*sintheta + yb2d*costheta, zb3d = zb1d;
    const R xc3d = -xb2d*costheta - yc2d*sintheta, yc3d = -xb2d*sintheta + yc2d*costheta, zc3d = zc1d;
    // step 5
    const R xa3 = t11*xa3d + t12*ya3d + t13*za3d, ya3 = t21*xa3d + t22*ya3d + t23*za3d, za3 = t31*xa3d + t32*ya3d + t33*za3d;
    const R xb3 = t11*xb3d + t12*yb3d + t13*zb3d, yb3 = t21*xb3d + t22*yb3d + t23*zb3d, zb3 = t31*xb3d + t32*yb3d + t33*zb3d;
    const R xc3 = t11*xc3d + t12*yc3d + t13*zc3d, yc3 = t21*xc3d + t22*yc3d + t23*zc3d, zc3 = t31*xc3d + t32*yc3d + t33*zc3d;
    d[0] = {xcom + xa3, ycom + ya3, zcom + za3};
    d[1] = {xcom + xb3 - xb0, ycom + yb3 - yb0, zcom + zb3 - zb0};
    d[2] = {xcom + xc3 - xc0, ycom + yc3 - yc0, zcom + zc3 - zc0};
}

// SETTLE, velocities (ReferenceSETTLEAlgorithm.cpp:197-244; general masses)
template <class R>
__device__ void settle_velocities(const V3<R>* x, V3<R>* v, const R* m) {
    V3<R> eAB = x[1]-x[0], eBC = x[2]-x[1], eCA = x[0]-x[2];
    eAB = eAB*rsqrt_r(dot(eAB, eAB)); eBC = eBC*rsqrt_r(dot(eBC, eBC)); eCA = eCA*rsqrt_r(dot(eCA, eCA));
    const R vAB = dot(v[1]-v[0], eAB), vBC = dot(v[2]-v[1], eBC), vCA = dot(v[0]-v[2], eCA);
    const R cA = -dot(eAB, eCA), cB = -dot(eAB, eBC), cC = -dot(eBC, eCA);
    const R s2A = 1-cA*cA, s2B = 1-cB*cB, s2C = 1-cC*cC;
    const R mA = m[0], mB = m[1], mC = m[2];
    const R mABCinv = R(1)/(mA*mB*mC);
    const R denom = (((s2A*mB+s2B*mA)*mC+(s2A*mB*mB+2*(cA*cB*cC+1)*mA*mB+s2B*mA*mA))*mC+s2C*mA*mB*(mA+mB))*mABCinv;
    const R tab = ((cB*cC*mA-cA*mB-cA*mC)*vCA + (cA*cC*mB-cB*mC-cB*mA)*vBC + (s2C*mA*mA*mB*mB*mABCinv+(mA+mB+mC))*vAB)/denom;
    const R tbc = ((cA*cB*mC-cC*mB-cC*mA)*vCA + (s2A*mB*mB*mC*mC*mABCinv+(mA+mB+mC))*vBC + (cA*cC*mB-cB*mA-cB*mC)*vAB)/denom;
    const R tca = ((s2B*mA*mA*mC*mC*mABCinv+(mA+mB+mC))*vCA + (cA*cB*mC-cC*mB-cC*mA)*vBC + (cB*cC*mA-cA*mB-cA*mC)*vAB)/denom;
    v[0] = v[0] + (eAB*tab - eCA*tca)*(R(1)/mA);
    v[1] = v[1] + (eBC*tbc - eAB*tab)*(R(1)/mB);
    v[2] = v[2] + (eCA*tca - eBC*tbc)*(R(1)/mC);
}

// SHAKE on a centre + n hydrogens, positions (deltas d relative to old positions x)
template <class R>
__device__ void shake_positions(const V3<R>* x, V3<R>* d, const R* invM, const R* dist, int n, R tol) {
    V3<R> rij[3]; R rij2[3], ld[3];
    _Pragma("unroll") for (int k = 0; k < 3; k++) if (k < n) {
        rij[k] = x[0] - x[k+1];
        rij2[k] = dot(rij[k], rij[k]);
        ld[k] = dist[k]*dist[k] - rij2[k];
    }
    bool converged = false;
    for (int it = 0; it < 30 && !converged; it++) {
        converged = true;
        _Pragma("unroll") for (int k = 0; k < 3; k++) if (k < n) {
            const V3<R> rp = d[0] - d[k+1];
            const R rp2 = dot(rp, rp), rrpr = dot(rij[k], rp);
            const R diff = ld[k] - R(2)*rrpr - rp2;
            const R d2 = dist[k]*dist[k];
            if (fabs_r(diff) >= d2*tol) {
                const R acor = diff*R(0.5)/((invM[0] + invM[k+1])*(rrpr + rij2[k]));
                d[0] = d[0] + rij[k]*(acor*invM[0]);
                d[k+1] = d[k+1] - rij[k]*(acor*invM[k+1]);
                converged = false;
            }
        }
    }
}

template <class R>
__device__ void shake_velocities(const V3<R>* x, V3<R>* v, const R* invM, int n, R tol) {
    V3<R> rij[3]; R rij2[3];
    _Pragma("unroll") for (int k = 0; k < 3; k++) if (k < n) { rij[k] = x[0] - x[k+1]; rij2[k] = dot(rij[k], rij[k]); }
    bool converged = false;
    for (int it = 0; it < 30 && !converged; it++) {
        converged = true;
        _Pragma("unroll") for (int k = 0; k < 3; k++) if (k < n) {
            const V3<R> rp = v[0] - v[k+1];
            const R rrpr = dot(rp, rij[k]);
            const R delta = -rrpr/((invM[0] + invM[k+1])*rij2[k]);
            v[0] = v[0] + rij[k]*(delta*invM[0]);
            v[k+1] = v[k+1] - rij[k]*(delta*invM[k+1]);
            if (fabs_r(delta) > tol) converged = false;
        }
    }
}

template <class R>
struct Unit {
    int n;             // atoms in the unit
    int atom[4];
    int type;
    V3<R> x[4], v[4], f[4];
    R invM[4], m[4];
    R4<R> prm;
};

template <class R> __device__ R4<R> unit_params(const UnitDev& un, int u);
template <> __device__ __forceinline__ float4 unit_params<float>(const UnitDev& un, int u) { return un.unitParams[u]; }
template <> __device__ __forceinline__ double4 unit_params<double>(const UnitDev& un, int u) { return un.unitParamsD[u]; }

template <class R>
__device__ __forceinline__ void load_unit(const NbDev& nb, const UnitDev& un, int u, Unit<R>& U, bool wantForce) {
    const int4 at = un.unitAtoms[u];
    U.atom[0] = at.x; U.atom[1] = at.y; U.atom[2] = at.z; U.atom[3] = at.w;
    U.type = un.unitType[u];
    U.prm = unit_params<R>(un, u);
    U.n = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int a = U.atom[k];
        if (a < 0) continue;
        U.n = k+1;
        const R4<R> p = load_pos<R>(nb, a);
        const R4<R> v = vel_array<R>(nb)[a];
        U.x[k] = {p.x, p.y, p.z};
        U.v[k] = {v.x, v.y, v.z};
        U.invM[k] = v.w;
        U.m[k] = (v.w > R(0)) ? R(1)/v.w : R(0);
        if (wantForce) {
            const long long fx = nb.force[a], fy = nb.force[a + nb.npad], fz = nb.force[a + 2*nb.npad];
            U.f[k] = {fixed_to_real<R>(fx), fixed_to_real<R>(fy), fixed_to_real<R>(fz)};
        }
    }
}

template <class R>
__device__ __forceinline__ void constrain_pos(const Unit<R>& U, V3<R>* d, R tol) {
    if (U.type == 1) settle_positions(U.x, d, U.m, U.prm.x, U.prm.y);
    else if (U.type == 2) { const R dist[3] = {U.prm.x, U.prm.y, U.prm.z}; shake_positions(U.x, d, U.invM, dist, U.n-1, tol); }
}
template <class R>
__device__ __forceinline__ void constrain_vel(const Unit<R>& U, V3<R>* v, R tol) {
    if (U.type == 1) settle_velocities(U.x, v, U.m);
    else if (U.type == 2) shake_velocities(U.x, v, U.invM, U.n-1, tol);
}

// Work mapping of k_integrate: 4 lanes per unit, lane k of the group owns atom k of the unit (lanes past the unit's atom
// count only join the shuffles).  Loads, force zeroing, CM-velocity removal, noise, the velocity update and the stores are
// per atom; for the constraint solve every lane of the group gathers the whole unit by warp shuffle and runs the same
// SETTLE / SHAKE code on the same operands (so all four hold the same bits) and keeps its own atom's result.  A group never
// straddles a warp (8 units per warp).  A block covers INTEG_UNITS units, the same 64 as the one-thread-per-unit kernel it
// replaced, so its centre-of-mass partial is summed over the same units in the same order.
constexpr int INTEG_LANES = 4;
constexpr int INTEG_UNITS = 64;
constexpr int INTEG_THREADS = INTEG_LANES*INTEG_UNITS;

__device__ __forceinline__ float shfl_r(float x, int src) { return __shfl_sync(0xffffffffu, x, src); }
__device__ __forceinline__ double shfl_r(double x, int src) { return __shfl_sync(0xffffffffu, x, src); }
template <class R>
__device__ __forceinline__ V3<R> shfl_v3(V3<R> a, int src) { return {shfl_r(a.x, src), shfl_r(a.y, src), shfl_r(a.z, src)}; }

// this lane's atom out of a per-unit array (unrolled selects: a dynamic index would put the array in local memory)
template <class T>
__device__ __forceinline__ T pick(const T* w, int k) {
    T r = w[0];
    _Pragma("unroll") for (int j = 1; j < 4; j++) if (k == j) r = w[j];
    return r;
}

// Fused epilogue work (in.fused != 0, the b200md_step path):
//  * centre-of-mass motion removal (CMMotionRemover, frequency 1): the momentum of the velocities this kernel WRITES is
//    reduced into cm[(step+1)%3]; the next step subtracts cm[step%3]/mass before integrating (same velocities, so the same
//    result as removing it at the start of that step, ReferenceKernels RemoveCMMotion); cm[(step+2)%3] is zeroed for reuse.
//  * the force buffer is zeroed after it has been read (saves the memset node at the head of the next step's graph).
//  * the last block to finish advances the step counter (saves a 1-thread kernel).
//
// Multi-GPU (cd.world > 1, single precision only): this rank integrates the units it OWNS.  The kernel first waits for the
// other ranks' partial forces (CH_FORCE), totals them with its own, and stores the new positions into EVERY rank's posq over
// NVLink -- the integrate step IS the position all-gather.  The last block hands its momentum sums to everybody and
// publishes CH_POS.
template <int KIND, class R>
__global__ void __launch_bounds__(INTEG_THREADS, 1) k_integrate(NbDev nb, UnitDev un, IntegDev in, CommDev cd) {
    const bool multi = cd.world > 1;
    const bool useInbox = multi && in.fused;       // step path; after b200md_compute the force buffer already holds the totals
    const unsigned long long E = multi ? *cd.epoch + 1ull : 0ull;
    if (useInbox) comm_wait(cd, CH_FORCE, E);
    const int ka = threadIdx.x & (INTEG_LANES - 1);                     // this lane's atom in its unit
    const int g = threadIdx.x & 31 & ~(INTEG_LANES - 1);               // the group's first lane in the warp
    const int ub = threadIdx.x / INTEG_LANES;                          // the unit's index in the block
    const int u = (multi ? cd.unitLo[cd.rank] : 0) + blockIdx.x*INTEG_UNITS + ub;
    const bool active = u < (multi ? cd.unitLo[cd.rank + 1] : un.nunits);
    const unsigned long long step = *in.stepCounter;
    const IntegR<R> ic = integ_r<R>(in);
    const R invDt = R(1)/ic.dt;
    const bool cmFused = in.fused && in.cmEveryStep;
    V3<R> vcm = {R(0), R(0), R(0)};
    if (cmFused) {
        double c[4];
        if (multi) {
            // every rank left the momentum of ITS atoms in slot [rank][step % 3] of everybody's table
            const double* t = (const double*) (cd.peer[cd.rank] + cd.offCm) + 4*(step % 3ull);
            c[0] = c[1] = c[2] = c[3] = 0.0;
            for (int q = 0; q < cd.world; q++) for (int k = 0; k < 4; k++) c[k] += t[q*12 + k];
        }
        else { const double* t = in.cmScratch + 4*(step % 3ull); c[0] = t[0]; c[1] = t[1]; c[2] = t[2]; c[3] = t[3]; }
        const double im = (c[3] > 0.0) ? 1.0/c[3] : 0.0;
        vcm = {(R) (c[0]*im), (R) (c[1]*im), (R) (c[2]*im)};
    }
    // the unit's constraint data (every lane of the group reads the same words) and this lane's atom
    Unit<R> U;
    U.n = 0; U.type = 0;
    int a = -1;
    if (active) {
        const int4 at = un.unitAtoms[u];
        U.n = at.w >= 0 ? 4 : at.z >= 0 ? 3 : at.y >= 0 ? 2 : at.x >= 0 ? 1 : 0;
        a = ka == 0 ? at.x : ka == 1 ? at.y : ka == 2 ? at.z : at.w;
        U.type = un.unitType[u];
        U.prm = unit_params<R>(un, u);
    }
    const bool own = a >= 0;
    V3<R> x = {R(0), R(0), R(0)}, v = x, f = x, d = x;
    R invM = R(0), m = R(0);
    if (own) {
        const R4<R> p = load_pos<R>(nb, a);
        const R4<R> vm = vel_array<R>(nb)[a];
        x = {p.x, p.y, p.z};
        v = {vm.x, vm.y, vm.z};
        invM = vm.w;
        m = (vm.w > R(0)) ? R(1)/vm.w : R(0);
        long long fx = nb.force[a], fy = nb.force[a + nb.npad], fz = nb.force[a + 2*nb.npad];
        if (useInbox) {
            // owner: total = own partial + what the other ranks pushed into the inboxes (exact int64 sums, any order)
            const long long* inbox = (const long long*) (cd.peer[cd.rank] + cd.offFinbox);
            for (int q = 0; q < cd.world; q++) if (q != cd.rank) {
                const long long* iq = inbox + (size_t) q*3*nb.npad;
                fx += iq[a]; fy += iq[a + nb.npad]; fz += iq[a + 2*nb.npad];
            }
        }
        f = {fixed_to_real<R>(fx), fixed_to_real<R>(fy), fixed_to_real<R>(fz)};
        if (in.fused) {
            nb.force[a] = 0; nb.force[a + nb.npad] = 0; nb.force[a + 2*nb.npad] = 0;
            if (invM > R(0)) v = v - vcm;
        }
    }
    // the group's old positions and masses for the solve (whole warps take part; a warp of free atoms skips it)
    const bool solve = __any_sync(0xffffffffu, U.type != 0);
    if (solve) {
        _Pragma("unroll") for (int j = 0; j < 4; j++) {
            U.x[j] = shfl_v3(x, g + j);
            U.invM[j] = shfl_r(invM, g + j);
            U.m[j] = shfl_r(m, g + j);
        }
    }
    V3<R> uw[4];
    if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
        if (own) v = v + f*(ic.dt*invM);
        if (solve) {
            _Pragma("unroll") for (int j = 0; j < 4; j++) uw[j] = shfl_v3(v, g + j);
            constrain_vel(U, uw, ic.tol);
            v = pick(uw, ka);
        }
        V3<R> du = d;
        if (own) {
            d = v*(R(0.5)*ic.dt);
            if (invM > R(0)) {
                const float3 gn = gauss3(in.seed, a, step);
                const R ns = ic.noisescale*sqrt_r(ic.kT*invM);
                v = v*ic.vscale + V3<R>{gn.x, gn.y, gn.z}*ns;
            }
            d = d + v*(R(0.5)*ic.dt);
            if (invM == R(0)) d = {R(0), R(0), R(0)};
            du = d;
        }
        if (solve) {
            _Pragma("unroll") for (int j = 0; j < 4; j++) uw[j] = shfl_v3(d, g + j);
            constrain_pos(U, uw, ic.tol);
            d = pick(uw, ka);
        }
        if (own) v = v + (d - du)*invDt;
    }
    else {
        if (own) {
            V3<R> vn;
            if (KIND == B200MD_INT_LANGEVIN) {
                vn = v*ic.vscale + f*(ic.fscale*invM);
                if (invM > R(0) && ic.noisescale > R(0)) {
                    const float3 gn = gauss3(in.seed, a, step);
                    vn = vn + V3<R>{gn.x, gn.y, gn.z}*(ic.noisescale*sqrt_r(invM));
                }
            }
            else
                vn = v + f*(ic.dt*invM);
            if (invM == R(0)) vn = v;
            d = (invM == R(0)) ? V3<R>{R(0), R(0), R(0)} : vn*ic.dt;
        }
        if (solve) {
            _Pragma("unroll") for (int j = 0; j < 4; j++) uw[j] = shfl_v3(d, g + j);
            constrain_pos(U, uw, ic.tol);
            d = pick(uw, ka);
        }
        if (own && invM > R(0)) v = d*invDt;
    }
    if (own) {
        store_pos<R>(nb, a, x.x + d.x, x.y + d.y, x.z + d.z);
        vel_array<R>(nb)[a] = make_r4(v.x, v.y, v.z, invM);
        if (multi && !cd.posByPush) {
            const float4 pn = nb.posq[a];
            for (int k = 1; k < cd.world; k++) {            // staggered: rank r starts with peer r+1, so the ranks do not all hit peer 0 first
                const int q = (cd.rank + k) % cd.world;
                ((float4*) (cd.peer[q] + cd.offPosq))[a] = pn;
            }
        }
    }
    if (!in.fused && !(multi && !cd.posByPush)) return;
    if (cmFused) {
        // the block's momentum sum, grouped as one thread per unit grouped it: per unit in atom order, a 32-unit xor
        // butterfly, then the sum of the 2 groups of 32 units
        // (the same px += mk*v form as there, so the compiler contracts it the same way)
        const bool mine = own && invM > R(0);
        double px = 0, py = 0, pz = 0, pm = 0;
        _Pragma("unroll") for (int j = 0; j < 4; j++) {
            const int cj = __shfl_sync(0xffffffffu, (int) mine, g + j);
            const double mk = shfl_r((double) m, g + j);
            const V3<R> vj = shfl_v3(v, g + j);
            if (cj) { px += mk*vj.x; py += mk*vj.y; pz += mk*vj.z; pm += mk; }
        }
        __shared__ double unitP[INTEG_UNITS][4];
        if (ka == 0) { unitP[ub][0] = px; unitP[ub][1] = py; unitP[ub][2] = pz; unitP[ub][3] = pm; }
        __shared__ double red[INTEG_UNITS/32][4];
        __syncthreads();
        if (threadIdx.x < INTEG_UNITS) {
            px = unitP[threadIdx.x][0]; py = unitP[threadIdx.x][1]; pz = unitP[threadIdx.x][2]; pm = unitP[threadIdx.x][3];
            for (int off = 16; off > 0; off >>= 1) {
                px += __shfl_xor_sync(0xffffffffu, px, off); py += __shfl_xor_sync(0xffffffffu, py, off);
                pz += __shfl_xor_sync(0xffffffffu, pz, off); pm += __shfl_xor_sync(0xffffffffu, pm, off);
            }
            if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = px; red[threadIdx.x >> 5][1] = py; red[threadIdx.x >> 5][2] = pz; red[threadIdx.x >> 5][3] = pm; }
        }
        __syncthreads();
        if (threadIdx.x < 4) {
            double t = 0;
            for (int w = 0; w < INTEG_UNITS/32; w++) t += red[w][threadIdx.x];
            atomicAdd(&in.cmScratch[4*((step + 1ull) % 3ull) + threadIdx.x], t);
            if (blockIdx.x == 0) in.cmScratch[4*((step + 2ull) % 3ull) + threadIdx.x] = 0.0;
        }
    }
    if (multi && !cd.posByPush) {
        // last block: momentum sums of this rank's atoms -> slot [rank][(step+1) % 3] of every rank's table, then CH_POS
        const bool lastBlock = comm_arrive(cd, CH_POS, gridDim.x);
        if (lastBlock && threadIdx.x == 0) {
            if (cmFused) {
                const double* mine = in.cmScratch + 4*((step + 1ull) % 3ull);
                for (int q = 0; q < cd.world; q++) {
                    double* t = (double*) (cd.peer[q] + cd.offCm) + cd.rank*12 + 4*((step + 1ull) % 3ull);
                    for (int k = 0; k < 4; k++) t[k] = ((volatile const double*) mine)[k];
                }
            }
            comm_publish(cd, CH_POS, E);
            *cd.posNeed = E;
            *cd.epoch = E;
            *in.stepCounter = step + 1ull;
        }
        return;
    }
    // last block to finish: advance the step counter
    __shared__ int last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        last = (atomicAdd(in.blocksDone, 1u) == gridDim.x - 1);
    }
    __syncthreads();
    if (last && threadIdx.x == 0) {
        *in.blocksDone = 0u;
        *in.stepCounter = step + 1ull;
    }
}

__global__ void k_step_advance(IntegDev in) { *in.stepCounter += 1ull; }

// momentum of the current velocities into cm[step % 3] (validates the fused scheme after the state was set from outside)
template <class R>
__global__ void __launch_bounds__(256) k_cm_prime(NbDev nb, IntegDev in, double* table) {
    const unsigned long long step = *in.stepCounter;
    double* c = table + 4*(step % 3ull);
    const int a = blockIdx.x*blockDim.x + threadIdx.x;
    double px = 0, py = 0, pz = 0, m = 0;
    if (a < nb.natoms) {
        const R4<R> v = vel_array<R>(nb)[a];
        if (v.w > R(0)) { m = 1.0/v.w; px = m*v.x; py = m*v.y; pz = m*v.z; }
    }
    for (int off = 16; off > 0; off >>= 1) {
        px += __shfl_xor_sync(0xffffffffu, px, off); py += __shfl_xor_sync(0xffffffffu, py, off);
        pz += __shfl_xor_sync(0xffffffffu, pz, off); m += __shfl_xor_sync(0xffffffffu, m, off);
    }
    __shared__ double red[8][4];
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = px; red[threadIdx.x >> 5][1] = py; red[threadIdx.x >> 5][2] = pz; red[threadIdx.x >> 5][3] = m; }
    __syncthreads();
    if (threadIdx.x < 4) {
        double t = 0;
        for (int w = 0; w < 8; w++) t += red[w][threadIdx.x];
        atomicAdd(&c[threadIdx.x], t);
    }
}

// Multi-GPU: the velocities are in sync at this point (the caller ran launch_vel_push), every rank computes the same total
// over ALL atoms and leaves it in row 0 of its own table (the other rows zero): k_integrate sums the rows.
void launch_cm_prime(const NbDev& nb, const IntegDev& integ, const CommDev& cd, cudaStream_t s) {
    cudaMemsetAsync(integ.cmScratch, 0, 12*sizeof(double), s);
    double* table = integ.cmScratch;
    if (cd.world > 1) {
        table = (double*) (cd.peer[cd.rank] + cd.offCm);
        cudaMemsetAsync(table, 0, (size_t) B200MD_MAX_RANKS*12*sizeof(double), s);
    }
    if (nb.velmD) k_cm_prime<double><<<(nb.natoms + 255)/256, 256, 0, s>>>(nb, integ, table);
    else k_cm_prime<float><<<(nb.natoms + 255)/256, 256, 0, s>>>(nb, integ, table);
}

template <int KIND>
static void launch_integrate_kind(int grid, const NbDev& nb, const UnitDev& units, const IntegDev& integ, const CommDev& cd, cudaStream_t s) {
    if (nb.velmD) k_integrate<KIND, double><<<grid, INTEG_THREADS, 0, s>>>(nb, units, integ, cd);
    else k_integrate<KIND, float><<<grid, INTEG_THREADS, 0, s>>>(nb, units, integ, cd);
}

void launch_integrate(const NbDev& nb, const UnitDev& units, const IntegDev& integ, const CommDev& cd, cudaStream_t s) {
    // 64 units (256 threads) per block: DHFR's 8k units give 128 blocks of 8 warps, one per SM of an H100 (132)
    const int n = cd.world > 1 ? cd.unitLo[cd.rank + 1] - cd.unitLo[cd.rank] : units.nunits;
    const int grid = std::max(1, (n + INTEG_UNITS - 1)/INTEG_UNITS);
    if (integ.kind == B200MD_INT_VERLET) launch_integrate_kind<B200MD_INT_VERLET>(grid, nb, units, integ, cd, s);
    else if (integ.kind == B200MD_INT_LANGEVIN) launch_integrate_kind<B200MD_INT_LANGEVIN>(grid, nb, units, integ, cd, s);
    else launch_integrate_kind<B200MD_INT_LANGEVIN_MIDDLE>(grid, nb, units, integ, cd, s);
    if (!integ.fused && (cd.world <= 1 || cd.posByPush)) k_step_advance<<<1, 1, 0, s>>>(integ);
    // multi-GPU, posByPush: the new positions of the owned atoms (one contiguous range) go to every peer through the TMA
    // engine in a kernel of their own, which also carries the momentum sums and publishes CH_POS
    if (cd.world > 1 && cd.posByPush) launch_pos_push(nb, cd, integ, s);
}

// ApplyConstraintsKernel::apply: project the current positions onto the constraints (reference & target identical)
template <class R>
__global__ void __launch_bounds__(128) k_constrain_positions(NbDev nb, UnitDev un, R tol) {
    const int u = blockIdx.x*blockDim.x + threadIdx.x;
    if (u >= un.nunits) return;
    Unit<R> U;
    load_unit(nb, un, u, U, false);
    if (U.type == 0) return;
    V3<R> d[4] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    constrain_pos(U, d, tol);
    _Pragma("unroll") for (int k = 0; k < 4; k++) if (k < U.n) {
        const int a = U.atom[k];
        const R4<R> p = load_pos<R>(nb, a);
        store_pos<R>(nb, a, p.x + d[k].x, p.y + d[k].y, p.z + d[k].z);
    }
}

template <class R>
__global__ void __launch_bounds__(128) k_constrain_velocities(NbDev nb, UnitDev un, R tol) {
    const int u = blockIdx.x*blockDim.x + threadIdx.x;
    if (u >= un.nunits) return;
    Unit<R> U;
    load_unit(nb, un, u, U, false);
    if (U.type == 0) return;
    constrain_vel(U, U.v, tol);
    _Pragma("unroll") for (int k = 0; k < 4; k++) if (k < U.n) vel_array<R>(nb)[U.atom[k]] = make_r4(U.v[k].x, U.v[k].y, U.v[k].z, U.invM[k]);
}

void launch_constrain_positions(const NbDev& nb, const UnitDev& units, double tol, cudaStream_t s) {
    if (units.nunits == 0) return;          // every atom sits in a general constraint network (constraints.cu)
    if (nb.velmD) k_constrain_positions<double><<<(units.nunits + 127)/128, 128, 0, s>>>(nb, units, tol);
    else k_constrain_positions<float><<<(units.nunits + 127)/128, 128, 0, s>>>(nb, units, (float) tol);
}
void launch_constrain_velocities(const NbDev& nb, const UnitDev& units, double tol, cudaStream_t s) {
    if (units.nunits == 0) return;
    if (nb.velmD) k_constrain_velocities<double><<<(units.nunits + 127)/128, 128, 0, s>>>(nb, units, tol);
    else k_constrain_velocities<float><<<(units.nunits + 127)/128, 128, 0, s>>>(nb, units, (float) tol);
}

// kinetic energy at time-shifted, re-constrained velocities (computeShiftedKineticEnergy, ReferenceKernels.cpp:146-176)
template <class R>
__global__ void __launch_bounds__(128) k_kinetic_energy(NbDev nb, UnitDev un, R shiftDt) {
    const int u = blockIdx.x*blockDim.x + threadIdx.x;
    double ke = 0.0;
    if (u < un.nunits) {
        Unit<R> U;
        load_unit(nb, un, u, U, true);
        if (shiftDt != R(0)) {
            _Pragma("unroll") for (int k = 0; k < 4; k++) if (k < U.n) U.v[k] = U.v[k] + U.f[k]*(shiftDt*U.invM[k]);
            constrain_vel(U, U.v, R(1e-4f));
        }
        _Pragma("unroll") for (int k = 0; k < 4; k++) if (k < U.n) ke += 0.5*(double) U.m[k]*(double) dot(U.v[k], U.v[k]);
    }
    for (int off = 16; off > 0; off >>= 1) ke += __shfl_xor_sync(0xffffffffu, ke, off);
    __shared__ double red[4];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ke;
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(&nb.energy[EN_KE], red[0] + red[1] + red[2] + red[3]);
}

void launch_kinetic_energy(const NbDev& nb, const UnitDev& units, const IntegDev& integ, double shiftDt, cudaStream_t s) {
    (void) integ;
    if (units.nunits == 0) return;
    if (nb.velmD) k_kinetic_energy<double><<<(units.nunits + 127)/128, 128, 0, s>>>(nb, units, shiftDt);
    else k_kinetic_energy<float><<<(units.nunits + 127)/128, 128, 0, s>>>(nb, units, (float) shiftDt);
}

// CMMotionRemover (ReferenceKernels.cpp RemoveCMMotion): subtract the centre-of-mass velocity.
template <class R>
__global__ void __launch_bounds__(256) k_cm_sum(NbDev nb, double* scratch) {
    const int a = blockIdx.x*blockDim.x + threadIdx.x;
    double px = 0, py = 0, pz = 0, m = 0;
    if (a < nb.natoms) {
        const R4<R> v = vel_array<R>(nb)[a];
        if (v.w > R(0)) { m = 1.0/v.w; px = m*v.x; py = m*v.y; pz = m*v.z; }
    }
    for (int off = 16; off > 0; off >>= 1) {
        px += __shfl_xor_sync(0xffffffffu, px, off); py += __shfl_xor_sync(0xffffffffu, py, off);
        pz += __shfl_xor_sync(0xffffffffu, pz, off); m += __shfl_xor_sync(0xffffffffu, m, off);
    }
    __shared__ double red[8][4];
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5][0] = px; red[threadIdx.x >> 5][1] = py; red[threadIdx.x >> 5][2] = pz; red[threadIdx.x >> 5][3] = m; }
    __syncthreads();
    if (threadIdx.x < 4) {
        double t = 0;
        for (int w = 0; w < 8; w++) t += red[w][threadIdx.x];
        atomicAdd(&scratch[threadIdx.x], t);
    }
}
template <class R>
__global__ void k_cm_apply(NbDev nb, double* scratch) {
    const int a = blockIdx.x*blockDim.x + threadIdx.x;
    if (a >= nb.natoms) return;
    const double im = 1.0/scratch[3];
    R4<R> v = vel_array<R>(nb)[a];
    if (v.w > R(0)) {
        v.x -= (R) (scratch[0]*im); v.y -= (R) (scratch[1]*im); v.z -= (R) (scratch[2]*im);
        vel_array<R>(nb)[a] = v;
    }
}
void launch_remove_cm(const NbDev& nb, double* scratch, cudaStream_t s) {
    cudaMemsetAsync(scratch, 0, 4*sizeof(double), s);
    if (nb.velmD) {
        k_cm_sum<double><<<(nb.natoms + 255)/256, 256, 0, s>>>(nb, scratch);
        k_cm_apply<double><<<(nb.natoms + 255)/256, 256, 0, s>>>(nb, scratch);
    }
    else {
        k_cm_sum<float><<<(nb.natoms + 255)/256, 256, 0, s>>>(nb, scratch);
        k_cm_apply<float><<<(nb.natoms + 255)/256, 256, 0, s>>>(nb, scratch);
    }
}

// ApplyMonteCarloBarostatKernel::scaleCoordinates (kernels.h:1425-1459) as ReferenceMonteCarloBarostat::applyBarostat does it
// (ReferenceMonteCarloBarostat.cpp:67-103): the unweighted centre of each barostat molecule, in user coordinates (positions
// plus cellOffset lattice vectors of the CURRENT box), is moved into the first periodic box (floor order c, b, a; origin 0),
// scaled, and every atom of the molecule moves by the same offset.  The positions receive the result in the working type (fp32,
// or hi + lo in mixed precision) and cellOffset becomes zero.
// One warp per molecule: lane l sums the atoms l, l+32, ... in double and an xor butterfly joins the lanes.  Addition is
// commutative, so every lane ends with the same bits and the result does not depend on scheduling: no atomics, two runs are
// bit-identical, and a 2,500-atom protein costs ~80 loads per lane instead of 2,500 on one thread.
template <class R>
__global__ void __launch_bounds__(256) k_scale_molecules(NbDev nb, ScaleDev sc) {
    const int m = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (m >= sc.nmol) return;                       // whole warps only: blockDim is a multiple of 32
    const int begin = sc.molStart[m], end = sc.molStart[m + 1];
    const int NP = nb.npad;
    double cx = 0, cy = 0, cz = 0;
    for (int t = begin + lane; t < end; t += 32) {
        const int a = sc.molAtoms[t];
        const R4<R> p = load_pos<R>(nb, a);
        const int kx = nb.cellOffset[a], ky = nb.cellOffset[a + NP], kz = nb.cellOffset[a + 2*NP];
        cx += (double) p.x + (kx*sc.a[0] + ky*sc.b[0] + kz*sc.c[0]);
        cy += (double) p.y + (ky*sc.b[1] + kz*sc.c[1]);
        cz += (double) p.z + kz*sc.c[2];
    }
    for (int off = 16; off > 0; off >>= 1) {
        cx += __shfl_xor_sync(0xffffffffu, cx, off); cy += __shfl_xor_sync(0xffffffffu, cy, off); cz += __shfl_xor_sync(0xffffffffu, cz, off);
    }
    const double inv = 1.0/(end - begin);           // Vec3::operator/= multiplies by the reciprocal
    cx *= inv; cy *= inv; cz *= inv;
    double x = cx, y = cy, z = cz, f;
    f = floor(z/sc.c[2]); x -= sc.c[0]*f; y -= sc.c[1]*f; z -= sc.c[2]*f;
    f = floor(y/sc.b[1]); x -= sc.b[0]*f; y -= sc.b[1]*f;
    f = floor(x/sc.a[0]); x -= sc.a[0]*f;
    const double ox = x*sc.s[0] - cx, oy = y*sc.s[1] - cy, oz = z*sc.s[2] - cz;
    for (int t = begin + lane; t < end; t += 32) {
        const int a = sc.molAtoms[t];
        const R4<R> p = load_pos<R>(nb, a);
        const int kx = nb.cellOffset[a], ky = nb.cellOffset[a + NP], kz = nb.cellOffset[a + 2*NP];
        const double ux = (double) p.x + (kx*sc.a[0] + ky*sc.b[0] + kz*sc.c[0]);
        const double uy = (double) p.y + (ky*sc.b[1] + kz*sc.c[1]);
        const double uz = (double) p.z + kz*sc.c[2];
        store_pos<R>(nb, a, (R) (ux + ox), (R) (uy + oy), (R) (uz + oz));
        nb.cellOffset[a] = 0; nb.cellOffset[a + NP] = 0; nb.cellOffset[a + 2*NP] = 0;
    }
}
void launch_scale_molecules(const NbDev& nb, const ScaleDev& sc, cudaStream_t s) {
    if (sc.nmol == 0) return;
    if (nb.velmD) k_scale_molecules<double><<<(sc.nmol + 7)/8, 256, 0, s>>>(nb, sc);
    else k_scale_molecules<float><<<(sc.nmol + 7)/8, 256, 0, s>>>(nb, sc);
}
