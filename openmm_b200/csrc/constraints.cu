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


// Block-wide CCMA solve of component `comp`.  VEL = false: positions `tgt` (new) against reference geometry xref (old,
// constraints satisfied); VEL = true: velocities `tgt` against the current geometry xref.  Both arrays are indexed by
// user atom.  Returns the number of iterations used (all threads).
template <bool VEL>
__device__ int ccma_solve(const CcmaDev& cc, int comp, float4* tgt, const float4* xref, const float4* velm, float tol) {
    const int c0 = cc.compConStart[comp], c1 = cc.compConStart[comp+1];
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    for (int k = c0 + threadIdx.x; k < c1; k += blockDim.x) {
        const int2 at = cc.conAtoms[k];
        const float4 pi = xref[at.x], pj = xref[at.y];
        const float dx = pi.x - pj.x, dy = pi.y - pj.y, dz = pi.z - pj.z;
        cc.rij[k] = make_float4(dx, dy, dz, dx*dx + dy*dy + dz*dz);
    }
    __syncthreads();
    const float lowerTol = 1.f - 2.f*tol + tol*tol, upperTol = 1.f + 2.f*tol + tol*tol;
    int iter = 0;
    for (; iter < cc.maxIter; iter++) {
        int converged = 1;
        for (int k = c0 + threadIdx.x; k < c1; k += blockDim.x) {
            const int2 at = cc.conAtoms[k];
            const float4 r = cc.rij[k];
            const float4 pi = tgt[at.x], pj = tgt[at.y];
            const float rx = pi.x - pj.x, ry = pi.y - pj.y, rz = pi.z - pj.z;
            const float rrpr = rx*r.x + ry*r.y + rz*r.z;
            float delta;
            if (VEL) {
                delta = -2.f*cc.conRedMass[k]*rrpr/r.w;
                if (!(fabsf(delta) <= tol)) converged = 0;
            }
            else {
                const float rp2 = rx*rx + ry*ry + rz*rz;
                const float d2 = cc.conDist[k]*cc.conDist[k];
                delta = cc.conRedMass[k]*(d2 - rp2)/rrpr;
                if (!(rp2 >= lowerTol*d2 && rp2 <= upperTol*d2)) converged = 0;
            }
            cc.delta1[k] = delta;
        }
        if (__syncthreads_and(converged)) break;
        // delta2 = (approximate inverse of the coupling matrix) * delta1
        for (int k = c0 + threadIdx.x; k < c1; k += blockDim.x) {
            float sum = 0.f;
            for (int e = cc.rowStart[k]; e < cc.rowStart[k+1]; e++) sum += cc.val[e]*cc.delta1[cc.col[e]];
            cc.delta2[k] = sum;
        }
        __syncthreads();
        // every atom gathers the displacements of its constraints (no atomics: the result does not depend on thread order)
        for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
            const int a = cc.atoms[t];
            const float w = velm[a].w;
            float4 p = tgt[a];
            float sx = 0.f, sy = 0.f, sz = 0.f;
            for (int e = cc.aStart[t]; e < cc.aStart[t+1]; e++) {
                const int code = cc.aCon[e];
                const int k = (code > 0 ? code : -code) - 1;
                const float s = (code > 0 ? 1.f : -1.f)*cc.delta2[k];
                const float4 r = cc.rij[k];
                sx += s*r.x; sy += s*r.y; sz += s*r.z;
            }
            p.x += sx*w; p.y += sy*w; p.z += sz*w;
            tgt[a] = p;
        }
        __syncthreads();
    }
    return iter;
}

// One MD step of the atoms of one constraint component (the counterpart of k_integrate for them).
template <int KIND>
__global__ void __launch_bounds__(256) k_ccma_step(NbDev nb, CcmaDev cc, IntegDev in) {
    const int comp = blockIdx.x;
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    const unsigned long long step = *in.stepCounter;
    const bool cmFused = in.fused && in.cmEveryStep;
    float vcx = 0.f, vcy = 0.f, vcz = 0.f;
    if (cmFused) {
        const double* c = in.cmScratch + 4*(step % 3ull);
        const double im = (c[3] > 0.0) ? 1.0/c[3] : 0.0;
        vcx = (float) (c[0]*im); vcy = (float) (c[1]*im); vcz = (float) (c[2]*im);
    }
    const float invDt = 1.0f/in.dt;
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const int a = cc.atoms[t];
        const float4 p = nb.posq[a];
        float4 v = nb.velm[a];
        const float fx = fixed_to_float(nb.force[a]), fy = fixed_to_float(nb.force[a + nb.npad]), fz = fixed_to_float(nb.force[a + 2*nb.npad]);
        if (in.fused) { nb.force[a] = 0; nb.force[a + nb.npad] = 0; nb.force[a + 2*nb.npad] = 0; }
        if (v.w > 0.f) { v.x -= vcx; v.y -= vcy; v.z -= vcz; }
        if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
            v.x += fx*in.dt*v.w; v.y += fy*in.dt*v.w; v.z += fz*in.dt*v.w;
            nb.velm[a] = v;
        }
        else {
            float vx, vy, vz;
            if (KIND == B200MD_INT_LANGEVIN) {
                vx = v.x*in.vscale + fx*in.fscale*v.w; vy = v.y*in.vscale + fy*in.fscale*v.w; vz = v.z*in.vscale + fz*in.fscale*v.w;
                if (v.w > 0.f && in.noisescale > 0.f) {
                    const float3 g = gauss3(in.seed, a, step);
                    const float ns = in.noisescale*sqrtf(v.w);
                    vx += g.x*ns; vy += g.y*ns; vz += g.z*ns;
                }
            }
            else { vx = v.x + fx*in.dt*v.w; vy = v.y + fy*in.dt*v.w; vz = v.z + fz*in.dt*v.w; }
            if (v.w == 0.f) { vx = vy = vz = 0.f; }
            cc.xold[a] = p;
            nb.posq[a] = make_float4(p.x + vx*in.dt, p.y + vy*in.dt, p.z + vz*in.dt, p.w);
        }
    }
    __syncthreads();
    if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
        ccma_solve<true>(cc, comp, nb.velm, nb.posq, nb.velm, in.tol);
        for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
            const int a = cc.atoms[t];
            const float4 p = nb.posq[a];
            float4 v = nb.velm[a];
            float dx = v.x*(0.5f*in.dt), dy = v.y*(0.5f*in.dt), dz = v.z*(0.5f*in.dt);
            if (v.w > 0.f) {
                const float3 g = gauss3(in.seed, a, step);
                const float ns = in.noisescale*sqrtf(in.kT*v.w);
                v.x = v.x*in.vscale + g.x*ns; v.y = v.y*in.vscale + g.y*ns; v.z = v.z*in.vscale + g.z*ns;
            }
            dx += v.x*(0.5f*in.dt); dy += v.y*(0.5f*in.dt); dz += v.z*(0.5f*in.dt);
            if (v.w == 0.f) { dx = dy = dz = 0.f; }
            cc.xold[a] = p;
            const float4 pn = make_float4(p.x + dx, p.y + dy, p.z + dz, p.w);
            cc.xunc[a] = pn;
            nb.posq[a] = pn;
            nb.velm[a] = v;
        }
        __syncthreads();
    }
    ccma_solve<false>(cc, comp, nb.posq, cc.xold, nb.velm, in.tol);
    double px = 0, py = 0, pz = 0, m = 0;
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const int a = cc.atoms[t];
        const float4 p = nb.posq[a];
        float4 v = nb.velm[a];
        if (v.w > 0.f) {
            if (KIND == B200MD_INT_LANGEVIN_MIDDLE) {
                const float4 u = cc.xunc[a];
                v.x += (p.x - u.x)*invDt; v.y += (p.y - u.y)*invDt; v.z += (p.z - u.z)*invDt;
            }
            else {
                const float4 o = cc.xold[a];
                v.x = (p.x - o.x)*invDt; v.y = (p.y - o.y)*invDt; v.z = (p.z - o.z)*invDt;
            }
            nb.velm[a] = v;
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
template <bool VEL>
__global__ void __launch_bounds__(256) k_ccma_apply(NbDev nb, CcmaDev cc, float tol) {
    const int comp = blockIdx.x;
    if (VEL) { ccma_solve<true>(cc, comp, nb.velm, nb.posq, nb.velm, tol); return; }
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) cc.xold[cc.atoms[t]] = nb.posq[cc.atoms[t]];
    __syncthreads();
    ccma_solve<false>(cc, comp, nb.posq, cc.xold, nb.velm, tol);
}

// kinetic energy of the CCMA atoms at time-shifted, re-constrained velocities (computeShiftedKineticEnergy,
// ReferenceKernels.cpp:146-176); the shifted velocities live in cc.xunc
__global__ void __launch_bounds__(256) k_ccma_kinetic(NbDev nb, CcmaDev cc, float shiftDt, float tol) {
    const int comp = blockIdx.x;
    const int a0 = cc.compAtomStart[comp], a1 = cc.compAtomStart[comp+1];
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const int a = cc.atoms[t];
        float4 v = nb.velm[a];
        v.x += fixed_to_float(nb.force[a])*shiftDt*v.w; v.y += fixed_to_float(nb.force[a + nb.npad])*shiftDt*v.w; v.z += fixed_to_float(nb.force[a + 2*nb.npad])*shiftDt*v.w;
        cc.xunc[a] = v;
    }
    __syncthreads();
    if (shiftDt != 0.f) ccma_solve<true>(cc, comp, cc.xunc, nb.posq, nb.velm, tol);
    double ke = 0.0;
    for (int t = a0 + threadIdx.x; t < a1; t += blockDim.x) {
        const float4 v = cc.xunc[cc.atoms[t]];
        if (v.w > 0.f) ke += 0.5*(1.0/(double) v.w)*((double) v.x*v.x + (double) v.y*v.y + (double) v.z*v.z);
    }
    for (int off = 16; off > 0; off >>= 1) ke += __shfl_xor_sync(0xffffffffu, ke, off);
    if ((threadIdx.x & 31) == 0 && ke != 0.0) atomicAdd(&nb.energy[EN_KE], ke);
}

void launch_ccma_step(const NbDev& nb, const CcmaDev& cc, const IntegDev& in, cudaStream_t s) {
    if (cc.ncomp == 0) return;
    if (in.kind == B200MD_INT_VERLET) k_ccma_step<B200MD_INT_VERLET><<<cc.ncomp, 256, 0, s>>>(nb, cc, in);
    else if (in.kind == B200MD_INT_LANGEVIN) k_ccma_step<B200MD_INT_LANGEVIN><<<cc.ncomp, 256, 0, s>>>(nb, cc, in);
    else k_ccma_step<B200MD_INT_LANGEVIN_MIDDLE><<<cc.ncomp, 256, 0, s>>>(nb, cc, in);
}
void launch_ccma_apply(const NbDev& nb, const CcmaDev& cc, bool velocities, float tol, cudaStream_t s) {
    if (cc.ncomp == 0) return;
    if (velocities) k_ccma_apply<true><<<cc.ncomp, 256, 0, s>>>(nb, cc, tol);
    else k_ccma_apply<false><<<cc.ncomp, 256, 0, s>>>(nb, cc, tol);
}
void launch_ccma_kinetic(const NbDev& nb, const CcmaDev& cc, float shiftDt, float tol, cudaStream_t s) {
    if (cc.ncomp == 0) return;
    k_ccma_kinetic<<<cc.ncomp, 256, 0, s>>>(nb, cc, shiftDt, tol);
}
