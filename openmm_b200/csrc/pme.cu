// pme.cu -- PME charge spreading, influence function and force interpolation (sm_90a).
//
// Restates pme_update_grid_index_and_fraction / pme_update_bsplines / pme_grid_spread_charge /
// pme_grid_interpolate_force / pme_calculate_bsplines_moduli (ReferencePME.cpp:98-193, 206-405, 617-713);
// replaces findAtomGridIndex / gridSpreadCharge / finishSpreadCharge / gridInterpolateForce of the
// reference GPU platforms (platforms/common/src/kernels/pme.cc:1-161, 506-606).  Order-5 cardinal B-splines,
// forward-only stencil with periodic wrap, charges carry sqrt(ONE_4PI_EPS0).
#include "engine.h"
#include <algorithm>

#define ORDER B200MD_PME_ORDER

// theta / dtheta for one axis, the recursion of pme_update_bsplines (ReferencePME.cpp:274-327)
// The weights are formed in DOUBLE: every charge interacts with its own spread image through them (a term of
// q^2 x ~25 x 138 kJ/mol/nm that only cancels if spreading and interpolation use the same, accurate weights); fp32 weights
// left a reciprocal-space force error of ~4e-4 kJ/mol/nm on every system, whatever the precision of the FFT
// (profiles/r02_parity_probe.md).  ~75 DFMA per atom and axis: nothing against the grid traffic.
typedef double wreal;
__device__ __forceinline__ void bspline(wreal dr, wreal* data, wreal* ddata) {
    data[ORDER-1] = 0.f;
    data[1] = dr;
    data[0] = 1.f - dr;
#pragma unroll
    for (int k = 3; k < ORDER; k++) {
        const wreal div = 1.f/(k - 1.f);
        data[k-1] = div*dr*data[k-2];
#pragma unroll
        for (int l = 1; l < k-1; l++)
            data[k-l-1] = div*((dr + l)*data[k-l-2] + (k - l - dr)*data[k-l-1]);
        data[0] = div*(1.f - dr)*data[0];
    }
    ddata[0] = -data[0];
#pragma unroll
    for (int k = 1; k < ORDER; k++) ddata[k] = data[k-1] - data[k];
    const wreal div = 1.f/(ORDER - 1);
    data[ORDER-1] = div*dr*data[ORDER-2];
#pragma unroll
    for (int l = 1; l < ORDER-1; l++)
        data[ORDER-l-1] = div*((dr + l)*data[ORDER-l-2] + (ORDER - l - dr)*data[ORDER-l-1]);
    data[0] = div*(1.f - dr)*data[0];
}

// grid index and fraction (ReferencePME.cpp:206-266); the fractional coordinate is formed in double so that the
// B-spline argument keeps full fp32 precision on 128-point grids
// returns false for a non-finite coordinate (the atom is skipped; the NaN shows up in the integrator instead of
// as an out-of-bounds grid access)
__device__ __forceinline__ bool grid_index(const float4& p, const NbDev& nb, const PmeDev& pme, int* idx, wreal* frac) {
    const double* R = nb.box.recip;
    const int n[3] = {pme.nx, pme.ny, pme.nz};
    bool ok = true;
#pragma unroll
    for (int d = 0; d < 3; d++) {
        double t = p.x*R[d] + p.y*R[3+d] + p.z*R[6+d];
        t = (t - floor(t))*n[d];
        ok = ok && (t >= 0.0) && (t <= (double) n[d]);
        int ti = (int) t;
        frac[d] = (wreal) (t - ti);
        idx[d] = (ti >= n[d]) ? ti - n[d] : ti;
    }
    return ok;
}

// 8 lanes per atom, lane ix < 5 owns one x-plane of the 5x5x5 stencil (25 grid points): five times more independent
// atomics / loads in flight per atom than the one-thread-per-atom form (both kernels are L2-latency bound at 24k atoms).
// Multi-GPU: every rank spreads the atoms it owns into its OWN full-size grid; k_grid_push then hands each x slab to its
// owner.  The kernel waits for the position stores of the last step first (it runs on the reciprocal-space stream,
// beside k_check_gather).
__global__ void __launch_bounds__(128) k_pme_spread(NbDev nb, PmeDev pme, CommDev cd) {
    comm_wait(cd, CH_POS, cd.world > 1 ? *cd.posNeed : 0ull);
    const int t = blockIdx.x*blockDim.x + threadIdx.x;
    int s, end;
    if (cd.world > 1) { s = cd.atomLo[cd.rank] + (t >> 3); end = cd.atomLo[cd.rank + 1]; }
    else { const int per = (nb.natoms + nb.world - 1)/nb.world; s = nb.rank*per + (t >> 3); end = min(nb.natoms, (nb.rank+1)*per); }
    const int ix = t & 7;
    if (s >= end || ix >= ORDER) return;
    // USER order and the user-order (never lattice-shifted) coordinate: reciprocal space then does not depend on the
    // neighbour list at all and runs concurrently with the list rebuild; the fractional position is formed in double, so
    // the grid index/fraction is exact for fp32 inputs wherever the atom sits relative to the primary cell
    const float4 p = nb.posq[s];
    if (p.w == 0.f) return;
    int idx[3];
    wreal fr[3];
    if (!grid_index(p, nb, pme, idx, fr)) return;
    wreal tx[ORDER], ty[ORDER], tz[ORDER], dd[ORDER];
    bspline(fr[0], tx, dd);
    bspline(fr[1], ty, dd);
    bspline(fr[2], tz, dd);
    wreal txi = tx[0];
#pragma unroll
    for (int k = 1; k < ORDER; k++) if (ix == k) txi = tx[k];
    int xi = idx[0] + ix; if (xi >= pme.nx) xi -= pme.nx;
    const wreal qx = (nb.chargeD != nullptr ? nb.chargeD[s] : (double) p.w)*txi;
#pragma unroll
    for (int iy = 0; iy < ORDER; iy++) {
        int yi = idx[1] + iy; if (yi >= pme.ny) yi -= pme.ny;
        const wreal qxy = qx*ty[iy];
        long long* row = pme.gridFixed + ((size_t) xi*pme.ny + yi)*pme.nz;
#pragma unroll
        for (int iz = 0; iz < ORDER; iz++) {
            int zi = idx[2] + iz; if (zi >= pme.nz) zi -= pme.nz;
            // integer accumulation: the grid (hence every force) is independent of the order of the atomics
            atomicAdd((unsigned long long*) (row + zi), (unsigned long long) __double2ll_rn(qxy*tz[iz]*4294967296.0));
        }
    }
}

// Multi-GPU: the owner interpolates the forces of its atoms from the potential grid that the slab owners have written
// into everybody's window (CH_POT).
__global__ void __launch_bounds__(128) k_pme_gather(NbDev nb, PmeDev pme, CommDev cd) {
    if (cd.world > 1) comm_wait(cd, CH_POT, *cd.epoch + 1ull);
    int s, end;
    if (cd.world > 1) { s = cd.atomLo[cd.rank] + blockIdx.x*blockDim.x + threadIdx.x; end = cd.atomLo[cd.rank + 1]; }
    else { const int per = (nb.natoms + nb.world - 1)/nb.world; s = nb.rank*per + blockIdx.x*blockDim.x + threadIdx.x; end = min(nb.natoms, (nb.rank+1)*per); }
    if (s >= end) return;
    const float4 p = nb.posq[s];
    if (p.w == 0.f) return;
    int idx[3];
    wreal fr[3];
    if (!grid_index(p, nb, pme, idx, fr)) return;
    wreal tx[ORDER], ty[ORDER], tz[ORDER], dx[ORDER], dy[ORDER], dz[ORDER];
    bspline(fr[0], tx, dx);
    bspline(fr[1], ty, dy);
    bspline(fr[2], tz, dz);
    wreal fx = 0.f, fy = 0.f, fz = 0.f;
    // The derivative weights sum to zero along their axis, so a constant added to the potential changes no force: take the
    // potential relative to the stencil's centre point.  |phi| is hundreds of kJ/mol/e, its variation over a stencil a few
    // tens: the fp32 sums below lose ~10x less (ApoA1: reciprocal-space force error 3.8e-4 -> see profiles/r02_parity_probe).
    float phi0;
    {
        int xc = idx[0] + 2; if (xc >= pme.nx) xc -= pme.nx;
        int yc = idx[1] + 2; if (yc >= pme.ny) yc -= pme.ny;
        int zc = idx[2] + 2; if (zc >= pme.nz) zc -= pme.nz;
        phi0 = __ldg(pme.grid + ((size_t) xc*pme.ny + yc)*pme.nz + zc);
    }
#pragma unroll
    for (int ix = 0; ix < ORDER; ix++) {
        int xi = idx[0] + ix; if (xi >= pme.nx) xi -= pme.nx;
#pragma unroll
        for (int iy = 0; iy < ORDER; iy++) {
            int yi = idx[1] + iy; if (yi >= pme.ny) yi -= pme.ny;
            const real* row = pme.grid + ((size_t) xi*pme.ny + yi)*pme.nz;
            wreal sz = 0.f, sdz = 0.f;
#pragma unroll
            for (int iz = 0; iz < ORDER; iz++) {
                int zi = idx[2] + iz; if (zi >= pme.nz) zi -= pme.nz;
                const float g = __ldg(row + zi) - phi0;
                sz += tz[iz]*g;
                sdz += dz[iz]*g;
            }
            fx += dx[ix]*ty[iy]*sz;
            fy += tx[ix]*dy[iy]*sz;
            fz += tx[ix]*ty[iy]*sdz;
        }
    }
    // ReferencePME.cpp:708-711 (triclinic-aware)
    const double* R = nb.box.recip;
    const double q = nb.chargeD != nullptr ? nb.chargeD[s] : (double) p.w;
    const double gx = (double) fx*pme.nx, gy = (double) fy*pme.ny, gz = (double) fz*pme.nz;
    const double Fx = -q*(gx*R[0]);
    const double Fy = -q*(gx*R[3] + gy*R[4]);
    const double Fz = -q*(gx*R[6] + gy*R[7] + gz*R[8]);
    const int a = s;
    atomicAdd((unsigned long long*) &nb.force[a], (unsigned long long) __double2ll_rn(Fx*B200MD_FORCE_SCALE));
    atomicAdd((unsigned long long*) &nb.force[a + nb.npad], (unsigned long long) __double2ll_rn(Fy*B200MD_FORCE_SCALE));
    atomicAdd((unsigned long long*) &nb.force[a + 2*nb.npad], (unsigned long long) __double2ll_rn(Fz*B200MD_FORCE_SCALE));
}

// influence function on the half-complex grid (pme_reciprocal_convolution, ReferencePME.cpp:409-514), computed in
// double once per box change.  eterm = exp(-pi^2 m^2/alpha^2) / (pi V m^2 bx by bz); the (0,0,0) term is zero
// (the reference skips it; its inverse transform is a constant and exerts no force).
__global__ void k_pme_eterm(NbDev nb, PmeDev pme) {
    const size_t total = (size_t) pme.nx*pme.ny*pme.nzc;
    const size_t i = (size_t) blockIdx.x*blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int kz = (int) (i % pme.nzc);
    const int ky = (int) ((i / pme.nzc) % pme.ny);
    const int kx = (int) (i / ((size_t) pme.nzc*pme.ny));
    if (kx == 0 && ky == 0 && kz == 0) { pme.eterm[i] = 0; return; }
    const double* R = nb.box.recip;
    const double mx = (kx < (pme.nx+1)/2) ? kx : kx - pme.nx;
    const double my = (ky < (pme.ny+1)/2) ? ky : ky - pme.ny;
    const double mz = (kz < (pme.nz+1)/2) ? kz : kz - pme.nz;
    const double mhx = mx*R[0];
    const double mhy = mx*R[3] + my*R[4];
    const double mhz = mx*R[6] + my*R[7] + mz*R[8];
    const double m2 = mhx*mhx + mhy*mhy + mhz*mhz;
    const double pi = 3.14159265358979323846;
    const double factor = pi*pi/(pme.alpha*pme.alpha);
    const double denom = m2*pi*nb.box.volume*pme.moduli[0][kx]*pme.moduli[1][ky]*pme.moduli[2][kz];
    pme.eterm[i] = (real) (exp(-factor*m2)/denom);
}

void launch_pme_eterm(const NbDev& nb, const PmeDev& pme, cudaStream_t s) {
    size_t total = (size_t) pme.nx*pme.ny*pme.nzc;
    k_pme_eterm<<<(unsigned) ((total + 255)/256), 256, 0, s>>>(nb, pme);
}

void launch_pme_spread(const NbDev& nb, const PmeDev& pme, const CommDev& cd, cudaStream_t s) {
    cudaMemsetAsync(pme.gridFixed, 0, sizeof(long long)*(size_t) pme.nx*pme.ny*pme.nz, s);
    const int per = cd.world > 1 ? cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank] : (nb.natoms + nb.world - 1)/nb.world;
    k_pme_spread<<<std::max(1, (per*8 + 127)/128), 128, 0, s>>>(nb, pme, cd);
}

void launch_pme_gather(const NbDev& nb, const PmeDev& pme, const CommDev& cd, cudaStream_t s) {
    const int per = cd.world > 1 ? cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank] : (nb.natoms + nb.world - 1)/nb.world;
    k_pme_gather<<<std::max(1, (per + 127)/128), 128, 0, s>>>(nb, pme, cd);
}
