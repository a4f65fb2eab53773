// constraints.cu -- general constraint networks (CCMA) on the device, one CTA per connected component (sm_90a).
//
// Restates ReferenceCCMAAlgorithm::applyConstraints (ReferenceCCMAAlgorithm.cpp:235-316: positions and velocities) for the
// constraints that are neither a rigid 3-atom molecule (SETTLE) nor an X-H_n cluster (SHAKE, both inside k_integrate):
// e.g. every bond of a protein under constraints=AllBonds.  The reference GPU platforms run this as four kernels per
// iteration over ALL constraints with a host check of a pinned convergence flag every few iterations
// (integrationUtilities.cc:559-800, IntegrationUtilities.cpp applyConstraintsImpl).  Here connected components of the
// constraint graph (molecules) are independent problems: one CTA takes a component through the WHOLE step -- velocity /
// position update of its atoms, every CCMA iteration (three phases separated by __syncthreads), final velocities -- so a
// step stays one launch, has no host involvement and replays inside the step graph.  The approximate inverse of the
// coupling matrix comes from the host (engine.cu: build_ccma).
#include "engine.h"
#include "../../include/b200md.h"
#include <algorithm>




// The kernels are templated on the working type R (float: single precision; double: mixed precision, engine.h).  In single
// precision the solver works on posq itself; in mixed precision on a double copy of the positions (CcmaDev::xposD) that the
// kernel loads from hi + lo and stores back as hi / lo.  CcmaWork<R> selects the constants and scratch of the working type.
template <class R> struct CcmaWork {
    const R* conDist; const R* conRedMass;
    R4<R>* rij; R* delta1; R* delta2;
    R4<R>* xold; R4<R>* xunc;
};
template <class R> __device__ CcmaWork<R> ccma_work(const CcmaDev& cc);
template <> __device__ __forceinline__ CcmaWork<float> ccma_work<float>(const CcmaDev& cc) {
    return {cc.conDist, cc.conRedMass, cc.rij, cc.delta1, cc.delta2, cc.xold, cc.xunc};
}
template <> __device__ __forceinline__ CcmaWork<double> ccma_work<double>(const CcmaDev& cc) {
    return {cc.conDistD, cc.conRedMassD, cc.rijD, cc.delta1D, cc.delta2D, cc.xoldD, cc.xuncD};
}
// the positions the solver moves
template <class R> __device__ R4<R>* ccma_positions(const NbDev& nb, const CcmaDev& cc);
template <> __device__ __forceinline__ float4* ccma_positions<float>(const NbDev& nb, const CcmaDev& cc) { return nb.posq; }
template <> __device__ __forceinline__ double4* ccma_positions<double>(const NbDev& nb, const CcmaDev& cc) { return cc.xposD; }
template <class R> __host__ __device__ constexpr bool is_mixed() { return sizeof(R) == sizeof(double); }

// Block-wide CCMA solve of component `comp`.  VEL = false: positions `tgt` (new) against reference geometry xref (old,
// constraints satisfied); VEL = true: velocities `tgt` against the current geometry xref.  Both arrays are indexed by
// user atom.  Returns the number of iterations used (all threads).
template <bool VEL, class R>
__device__ int ccma_solve(const CcmaDev& cc, const CcmaWork<R>& W, int comp, R4<R>* tgt, const R4<R>* xref, const R4<R>* velm, R tol) {
    const int c0 = cc.compConStart[comp], c1 = cc.compConStart[comp+1];
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    for (int k = c0 + threadIdx.x; k < c1; k += blockDim.x) {
        const int2 at = cc.conAtoms[k];
        const R4<R> pi = xref[at.x], pj = xref[at.y];
        const R dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
        W.rij[k] = make_r4(dx, dy, dz, dx*dx + dy*dy + dz*dz);
    }
    __syncthreads();
    // in the working type: at tol = 1e-10, fp32 would make both bounds exactly 1
    const R lowerTol = R(1) - R(2)*tol + tol*tol, upperTol = R(1) + R(2)*tol + tol*tol;
    int iter = 0;
    for (; iter < cc.maxIter; iter++) {
        int converged = 1;
        for (int k = c0 + threadIdx.x; k < c1; k += blockDim.x) {
            const int2 at = cc.conAtoms[k];
            const R4<R> r = W.rij[k];
            const R4<R> pi = tgt[at.x], pj = tgt[at.y];
            const R rx = pi.x - pj.x, ry = pi.y - pj.y, rz = pi.z - pj.z;
            const R rrpr = rx*r.x + ry*r.y + rz*r.z;
            R delta;
            if (VEL) {
                delta = -R(2)*W.conRedMass[k]*rrpr/r.w;
                if (!(fabs_r(delta) <= tol)) converged = 0;
            }
            else {
                const R rp2 = rx*rx + ry*ry + rz*rz;
                const R d2 = W.conDist[k]*W.conDist[k];
                delta = W.conRedMass[k]*(d2 - rp2)/rrpr;
                if (!(rp2 >= lowerTol*d2 && rp2 <= upperTol*d2)) converged = 0;
            }
            W.delta1[k] = delta;
        }
        if (__syncthreads_and(converged)) break;
        // delta2 = (approximate inverse of the coupling matrix) * delta1
        for (int k = c0 + threadIdx.x; k < c1; k += blockDim.x) {
            R sum = R(0);
            for (int e = cc.rowStart[k]; e < cc.rowStart[k+1]; e++) sum += (R) cc.val[e]*W.delta1[cc.col[e]];
            W.delta2[k] = sum;
        }
        __syncthreads();
        // every atom gathers the displacements of its constraints (no atomics: the result does not depend on thread order)
        for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
            const int a = cc.atoms[t];
            const R w = velm[a].w;
            R4<R> p = tgt[a];
            R sx = R(0), sy = R(0), sz = R(0);
            for (int e = cc.aStart[t]; e < cc.aStart[t+1]; e++) {
                const int code = cc.aCon[e];
                const int k = (code > 0 ? code : -code) - 1;
                const R s = (code > 0 ? R(1) : R(-1))*W.delta2[k];
                const R4<R> r = W.rij[k];
                sx += s*r.x; sy += s*r.y; sz += s*r.z;
            }
            p.x += sx*w; p.y += sy*w; p.z += sz*w;
            tgt[a] = p;
        }
        __syncthreads();
    }
    return iter;
}

// mixed precision: the solver's positions <- hi + lo (a no-op in single precision, where they are posq itself)
template <class R>
__device__ __forceinline__ void ccma_load_positions(const NbDev& nb, const CcmaDev& cc, int a0, int a1) {
    if (!is_mixed<R>()) return;
    R4<R>* X = ccma_positions<R>(nb, cc);
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) X[cc.atoms[t]] = load_pos<R>(nb, cc.atoms[t]);
}
// mixed precision: hi / lo <- the solver's positions (same threads as the solver's last gather: no barrier needed)
template <class R>
__device__ __forceinline__ void ccma_store_positions(const NbDev& nb, const CcmaDev& cc, int a0, int a1) {
    if (!is_mixed<R>()) return;
    const R4<R>* X = ccma_positions<R>(nb, cc);
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) { const int a = cc.atoms[t]; store_pos<R>(nb, a, X[a].x, X[a].y, X[a].z); }
}

// One MD step of the atoms of one constraint component (the counterpart of k_integrate for them).
template <int KIND, class R>
__global__ void __launch_bounds__(256) k_ccma_step(NbDev nb, CcmaDev cc, IntegDev in) {
    const int comp = blockIdx.x;
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    const unsigned long long step = *in.stepCounter;
    const bool cmFused = in.fused && in.cmEveryStep;
    const IntegR<R> ic = integ_r<R>(in);
    const CcmaWork<R> W = ccma_work<R>(cc);
    R4<R>* vel = vel_array<R>(nb);
    R4<R>* X = ccma_positions<R>(nb, cc);
    R vcx = R(0), vcy = R(0), vcz = R(0);
    if (cmFused) {
        const double* c = in.cmScratch + 4*(step % 3ull);
        const double im = (c[3] > 0.0) ? 1.0/c[3] : 0.0;
        vcx = (R) (c[0]*im); vcy = (R) (c[1]*im); vcz = (R) (c[2]*im);
    }
    const R invDt = R(1)/ic.dt;
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const int a = cc.atoms[t];
        const R4<R> p = load_pos<R>(nb, a);
        R4<R> v = vel[a];
        const R fx = fixed_to_real<R>(nb.force[a]), fy = fixed_to_real<R>(nb.force[a + nb.npad]), fz = fixed_to_real<R>(nb.force[a + 2*nb.npad]);
        if (in.fused) { nb.force[a] = 0; nb.force[a + nb.npad] = 0; nb.force[a + 2*nb.npad] = 0; }
        if (v.w > R(0)) { v.x -= vcx; v.y -= vcy; v.z -= vcz; }
        if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
            v.x += fx*ic.dt*v.w; v.y += fy*ic.dt*v.w; v.z += fz*ic.dt*v.w;
            vel[a] = v;
            if (is_mixed<R>()) X[a] = p;
        }
        else {
            R vx, vy, vz;
            if (KIND == B200MD_INT_LANGEVIN) {
                vx = v.x*ic.vscale + fx*ic.fscale*v.w; vy = v.y*ic.vscale + fy*ic.fscale*v.w; vz = v.z*ic.vscale + fz*ic.fscale*v.w;
                if (v.w > R(0) && ic.noisescale > R(0)) {
                    const float3 g = gauss3(in.seed, a, step);
                    const R ns = ic.noisescale*sqrt_r(v.w);
                    vx += g.x*ns; vy += g.y*ns; vz += g.z*ns;
                }
            }
            else { vx = v.x + fx*ic.dt*v.w; vy = v.y + fy*ic.dt*v.w; vz = v.z + fz*ic.dt*v.w; }
            if (v.w == R(0)) { vx = vy = vz = R(0); }
            W.xold[a] = p;
            X[a] = make_r4(p.x + vx*ic.dt, p.y + vy*ic.dt, p.z + vz*ic.dt, p.w);
        }
    }
    __syncthreads();
    if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
        ccma_solve<true, R>(cc, W, comp, vel, X, vel, ic.tol);
        for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
            const int a = cc.atoms[t];
            const R4<R> p = X[a];
            R4<R> v = vel[a];
            R dx = v.x*(R(0.5)*ic.dt), dy = v.y*(R(0.5)*ic.dt), dz = v.z*(R(0.5)*ic.dt);
            if (v.w > R(0)) {
                const float3 g = gauss3(in.seed, a, step);
                const R ns = ic.noisescale*sqrt_r(ic.kT*v.w);
                v.x = v.x*ic.vscale + g.x*ns; v.y = v.y*ic.vscale + g.y*ns; v.z = v.z*ic.vscale + g.z*ns;
            }
            dx += v.x*(R(0.5)*ic.dt); dy += v.y*(R(0.5)*ic.dt); dz += v.z*(R(0.5)*ic.dt);
            if (v.w == R(0)) { dx = dy = dz = R(0); }
            W.xold[a] = p;
            const R4<R> pn = make_r4(p.x + dx, p.y + dy, p.z + dz, p.w);
            W.xunc[a] = pn;
            X[a] = pn;
            vel[a] = v;
        }
        __syncthreads();
    }
    ccma_solve<false, R>(cc, W, comp, X, W.xold, vel, ic.tol);
    double px = 0, py = 0, pz = 0, m = 0;
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const int a = cc.atoms[t];
        const R4<R> p = X[a];
        R4<R> v = vel[a];
        if (is_mixed<R>()) store_pos<R>(nb, a, p.x, p.y, p.z);
        if (v.w > R(0)) {
            if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
                const R4<R> u = W.xunc[a];
                v.x += (p.x - u.x)*invDt; v.y += (p.y - u.y)*invDt; v.z += (p.z - u.z)*invDt;
            }
            else {
                const R4<R> o = W.xold[a];
                v.x = (p.x - o.x)*invDt; v.y = (p.y - o.y)*invDt; v.z = (p.z - o.z)*invDt;
            }
            vel[a] = v;
            const double mk = 1.0/v.w;
            px += mk*v.x; py += mk*v.y; pz += mk*v.z; m += mk;
        }
    }
    if (cmFused) {
        for (int off = 16; off > 0; off >>= 1) {
            px += __shfl_xor_sync(0xffffffffu, px, off); py += __shfl_xor_sync(0xffffffffu, py, off);
            pz += __shfl_xor_sync(0xffffffffu, pz, off); m += __shfl_xor_sync(0xffffffffu, m, off);
        }
        if ((threadIdx.x & 31) == 0 && m > 0.0) {
            double* c = in.cmScratch + 4*((step + 1ull) % 3ull);
            atomicAdd(c, px); atomicAdd(c + 1, py); atomicAdd(c + 2, pz); atomicAdd(c + 3, m);
        }
    }
}

// ApplyConstraintsKernel::apply / applyToVelocities for the CCMA atoms
template <bool VEL, class R>
__global__ void __launch_bounds__(256) k_ccma_apply(NbDev nb, CcmaDev cc, R tol) {
    const int comp = blockIdx.x;
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    const CcmaWork<R> W = ccma_work<R>(cc);
    R4<R>* vel = vel_array<R>(nb);
    R4<R>* X = ccma_positions<R>(nb, cc);
    if (VEL) {
        ccma_load_positions<R>(nb, cc, a0, a1);
        if (is_mixed<R>()) __syncthreads();
        ccma_solve<true, R>(cc, W, comp, vel, X, vel, tol);
    }
    else {
        for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) W.xold[cc.atoms[t]] = load_pos<R>(nb, cc.atoms[t]);
        ccma_load_positions<R>(nb, cc, a0, a1);
        __syncthreads();
        ccma_solve<false, R>(cc, W, comp, X, W.xold, vel, tol);
        ccma_store_positions<R>(nb, cc, a0, a1);
    }
}

// kinetic energy of the CCMA atoms at time-shifted, re-constrained velocities (computeShiftedKineticEnergy,
// ReferenceKernels.cpp:146-176); the shifted velocities live in xunc
template <class R>
__global__ void __launch_bounds__(256) k_ccma_kinetic(NbDev nb, CcmaDev cc, R shiftDt, R tol) {
    const int comp = blockIdx.x;
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    const CcmaWork<R> W = ccma_work<R>(cc);
    R4<R>* vel = vel_array<R>(nb);
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const int a = cc.atoms[t];
        R4<R> v = vel[a];
        v.x += fixed_to_real<R>(nb.force[a])*shiftDt*v.w; v.y += fixed_to_real<R>(nb.force[a + nb.npad])*shiftDt*v.w; v.z += fixed_to_real<R>(nb.force[a + 2*nb.npad])*shiftDt*v.w;
        W.xunc[a] = v;
    }
    ccma_load_positions<R>(nb, cc, a0, a1);
    __syncthreads();
    if (shiftDt != R(0)) ccma_solve<true, R>(cc, W, comp, W.xunc, ccma_positions<R>(nb, cc), vel, tol);
    double ke = 0.0;
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const R4<R> v = W.xunc[cc.atoms[t]];
        if (v.w > R(0)) ke += 0.5*(1.0/(double) v.w)*((double) v.x*v.x + (double) v.y*v.y + (double) v.z*v.z);
    }
    for (int off = 16; off > 0; off >>= 1) ke += __shfl_xor_sync(0xffffffffu, ke, off);
    if ((threadIdx.x & 31) == 0 && ke != 0.0) atomicAdd(&nb.energy[EN_KE], ke);
}

template <class R>
static void launch_ccma_step_r(const NbDev& nb, const CcmaDev& cc, const IntegDev& in, cudaStream_t s) {
    if (in.kind == B200MD_INT_VERLET) k_ccma_step<B200MD_INT_VERLET, R><<<cc.ncomp, 256, 0, s>>>(nb, cc, in);
    else if (in.kind == B200MD_INT_LANGEVIN) k_ccma_step<B200MD_INT_LANGEVIN, R><<<cc.ncomp, 256, 0, s>>>(nb, cc, in);
    else k_ccma_step<B200MD_INT_LANGEVIN_MIDDLE, R><<<cc.ncomp, 256, 0, s>>>(nb, cc, in);
}
void launch_ccma_step(const NbDev& nb, const CcmaDev& cc, const IntegDev& in, cudaStream_t s) {
    if (cc.ncomp == 0) return;
    if (nb.velmD) launch_ccma_step_r<double>(nb, cc, in, s);
    else launch_ccma_step_r<float>(nb, cc, in, s);
}
template <class R>
static void launch_ccma_apply_r(const NbDev& nb, const CcmaDev& cc, bool velocities, R tol, cudaStream_t s) {
    if (velocities) k_ccma_apply<true, R><<<cc.ncomp, 256, 0, s>>>(nb, cc, tol);
    else k_ccma_apply<false, R><<<cc.ncomp, 256, 0, s>>>(nb, cc, tol);
}
void launch_ccma_apply(const NbDev& nb, const CcmaDev& cc, bool velocities, double tol, cudaStream_t s) {
    if (cc.ncomp == 0) return;
    if (nb.velmD) launch_ccma_apply_r<double>(nb, cc, velocities, tol, s);
    else launch_ccma_apply_r<float>(nb, cc, velocities, (float) tol, s);
}
void launch_ccma_kinetic(const NbDev& nb, const CcmaDev& cc, double shiftDt, double tol, cudaStream_t s) {
    if (cc.ncomp == 0) return;
    if (nb.velmD) k_ccma_kinetic<double><<<cc.ncomp, 256, 0, s>>>(nb, cc, shiftDt, tol);
    else k_ccma_kinetic<float><<<cc.ncomp, 256, 0, s>>>(nb, cc, (float) shiftDt, (float) tol);
}
