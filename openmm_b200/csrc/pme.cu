// pme.cu -- PME charge spreading, influence function and force interpolation (sm_90a).
//
// Restates pme_update_grid_index_and_fraction / pme_update_bsplines / pme_grid_spread_charge /
// pme_grid_interpolate_force / pme_calculate_bsplines_moduli (ReferencePME.cpp:98-193, 206-405, 617-713);
// replaces findAtomGridIndex / gridSpreadCharge / finishSpreadCharge / gridInterpolateForce of the
// reference GPU platforms (platforms/common/src/kernels/pme.cc:1-161, 506-606).  Order-5 cardinal B-splines,
// forward-only stencil with periodic wrap, charges carry sqrt(ONE_4PI_EPS0).
#include "engine.h"
#include <algorithm>
#include <climits>
#include <stdexcept>

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

// Shared-memory brick of the brick spread (launch_pme_spread with PmeDev::brickAtoms > 0): the box of grid points that the
// stencils of one CTA's atoms touch.  Point (x, y, z) of the brick is grid point (org + (x, y, z)) mod n, z fastest.  A
// contribution reaches the same grid point, with the same value, as in the user-order kernel, and the grid is an int64 sum,
// so the regrouping changes no bit.
struct Brick {
    int ref[3];                  // grid index of the CTA's first contributing atom
    int org[3];                  // brick origin, unwrapped (may lie outside [0, n))
    int ext[3];                  // brick extent per axis
    // periodic difference idx - ref on axis d, folded into (-n/2, n/2]
    __device__ __forceinline__ int rel(const int* idx, int d, int n) const {
        int r = idx[d] - ref[d];
        if (2*r > n) r -= n; else if (2*r <= -n) r += n;
        return r;
    }
    // brick coordinates of the stencil origin idx of an atom of this CTA
    __device__ __forceinline__ int local(const int* idx, int d, int n) const { return ref[d] + rel(idx, d, n) - org[d]; }
    __device__ __forceinline__ int points() const { return ext[0]*ext[1]*ext[2]; }
    // grid index of brick coordinate u on axis d: org + u lies in (-n/2, 3n/2 + ORDER - 1), below 3n for n >= 3
    __device__ __forceinline__ int wrap(int d, int u, int n) const {
        int g = org[d] + u;
        if (g < 0) g += n;
        if (g >= n) g -= n;
        if (g >= n) g -= n;
        return g;
    }
};

// slot k of the current list's sorted order: the user atom, or -1 when it contributes nothing (padding, zero charge)
__device__ __forceinline__ int brick_atom(const NbDev& nb, const ListDev& L, int k, float4& p) {
    if (k >= nb.npad) return -1;
    const int a = L.sorig[k];
    if (a < 0 || a >= nb.natoms) return -1;
    p = nb.posq[a];
    return p.w == 0.f ? -1 : a;
}

// Block-wide: bounds of the stencils of slots [k0, k0 + count) (count <= blockDim.x).  Indices are taken relative to the
// first contributing atom with the periodic difference folded into (-n/2, n/2], so a run of atoms that straddles the
// periodic boundary still gets a small brick.  Returns false (to all threads) when no slot contributes.
__device__ __forceinline__ bool brick_bounds(const NbDev& nb, const PmeDev& pme, const ListDev& L, int k0, int count, Brick& B) {
    __shared__ int sFirst, sRef[3], sLo[3], sHi[3];
    const int n[3] = {pme.nx, pme.ny, pme.nz};
    if (threadIdx.x == 0) {
        sFirst = INT_MAX;
        for (int d = 0; d < 3; d++) { sLo[d] = INT_MAX; sHi[d] = INT_MIN; }
    }
    __syncthreads();
    int idx[3];
    wreal fr[3];
    float4 p;
    const bool ok = (int) threadIdx.x < count && brick_atom(nb, L, k0 + threadIdx.x, p) >= 0 && grid_index(p, nb, pme, idx, fr);
    if (ok) atomicMin(&sFirst, (int) threadIdx.x);
    __syncthreads();
    if (sFirst == INT_MAX) return false;
    if ((int) threadIdx.x == sFirst) for (int d = 0; d < 3; d++) sRef[d] = idx[d];
    __syncthreads();
    for (int d = 0; d < 3; d++) B.ref[d] = sRef[d];
    if (ok) {
        for (int d = 0; d < 3; d++) {
            const int r = B.rel(idx, d, n[d]);
            atomicMin(&sLo[d], r); atomicMax(&sHi[d], r);
        }
    }
    __syncthreads();
    for (int d = 0; d < 3; d++) { B.org[d] = B.ref[d] + sLo[d]; B.ext[d] = sHi[d] - sLo[d] + ORDER; }
    return true;
}

// 64-bit shared-memory add as two native 32-bit ATOMS.ADD with the carry of the low word moved into the high word: exact
// modulo 2^64 whatever the order.  atomicAdd(unsigned long long*) on shared memory compiles to a compare-and-swap loop
// (ATOMS.CAST.SPIN.64) on sm_90a, which retries whenever the atoms of one water hit the same point together.
__device__ __forceinline__ void shared_add_u64(unsigned long long* p, unsigned long long v) {
    unsigned int* w = (unsigned int*) p;
    const unsigned int lo = (unsigned int) v;
    const unsigned int old = atomicAdd(w, lo);
    atomicAdd(w + 1, (unsigned int) (v >> 32) + (old + lo < old ? 1u : 0u));
}

// One atom's x-plane ix of the stencil: into the global grid, or (BRICK) into the CTA's brick.
// integer accumulation: the grid (hence every force) is independent of the order of the atomics
template <bool BRICK>
__device__ __forceinline__ void spread_atom(const NbDev& nb, const PmeDev& pme, int a, const float4& p, int ix, unsigned long long* brick, const Brick& B) {
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
    const wreal qx = (nb.chargeD != nullptr ? nb.chargeD[a] : (double) p.w)*txi;
    if (BRICK) {
        unsigned long long* plane = brick + ((size_t) (B.local(idx, 0, pme.nx) + ix)*B.ext[1] + B.local(idx, 1, pme.ny))*B.ext[2] + B.local(idx, 2, pme.nz);
#pragma unroll
        for (int iy = 0; iy < ORDER; iy++) {
            const wreal qxy = qx*ty[iy];
#pragma unroll
            for (int iz = 0; iz < ORDER; iz++)
                shared_add_u64(plane + iy*B.ext[2] + iz, (unsigned long long) __double2ll_rn(qxy*tz[iz]*4294967296.0));
        }
        return;
    }
#pragma unroll
    for (int iy = 0; iy < ORDER; iy++) {
        int yi = idx[1] + iy; if (yi >= pme.ny) yi -= pme.ny;
        const wreal qxy = qx*ty[iy];
        long long* row = pme.gridFixed + ((size_t) xi*pme.ny + yi)*pme.nz;
#pragma unroll
        for (int iz = 0; iz < ORDER; iz++) {
            int zi = idx[2] + iz; if (zi >= pme.nz) zi -= pme.nz;
            atomicAdd((unsigned long long*) (row + zi), (unsigned long long) __double2ll_rn(qxy*tz[iz]*4294967296.0));
        }
    }
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
    spread_atom<false>(nb, pme, s, p, ix, nullptr, Brick());
}

// Brick path of the spread (one GPU, a list exists): a CTA of 256 threads takes pme.brickAtoms consecutive slots of the
// current list's sorted order, spatially compact, so their stencils fit a brick of a few thousand points.  The atoms go
// into the brick in shared memory; then each non-zero brick point is added to the grid with ONE global atomic, coalesced
// along z, instead of one per atom and stencil point.  A brick above pme.brickPoints (atoms that are not compact, e.g.
// a stale order after set_positions moved molecules by lattice vectors) spreads those atoms straight to global memory.
// The list must not flip while this runs: enqueue_forces forks the reciprocal-space stream after the list build.
// It keeps 256 threads although a CTA (20,480 registers) does not fit the slot one retiring tile-kernel CTA hands back:
// measured on an H100 (700 W), 128-thread CTAs that do fit made the spread 10 us longer on ApoA1 and both steps slower.
__global__ void __launch_bounds__(256) k_pme_spread_brick(NbDev nb, PmeDev pme) {
    extern __shared__ unsigned long long brick[];
    const ListDev& L = nb.list[nb.counters[CT_CUR] & 1];
    const int count = pme.brickAtoms, k0 = blockIdx.x*count;
    Brick B;
    if (!brick_bounds(nb, pme, L, k0, count, B)) return;
    const int npts = B.points();
    const bool fits = npts <= pme.brickPoints;
    if (fits) {
        for (int c = threadIdx.x; c < npts; c += blockDim.x) brick[c] = 0ull;
        __syncthreads();
    }
    const int ix = threadIdx.x & 7, g = threadIdx.x >> 3, ng = blockDim.x >> 3;
    // the four atoms of a warp are ng/4 slots apart: consecutive slots (the atoms of one water) hit the same points
    const int perm = (g & 3)*(ng >> 2) + (g >> 2);
    for (int j = 0; j < count; j += ng) {
        float4 p;
        const int a = (j + perm < count && ix < ORDER) ? brick_atom(nb, L, k0 + j + perm, p) : -1;
        if (a < 0) continue;
        if (fits) spread_atom<true>(nb, pme, a, p, ix, brick, B);
        else spread_atom<false>(nb, pme, a, p, ix, nullptr, B);
    }
    if (!fits) return;
    __syncthreads();
    // consecutive threads take consecutive points (coalesced along z); each thread steps its (x, y, z) by blockDim.x points
    // with carries instead of dividing per point
    int z = threadIdx.x % B.ext[2], y = threadIdx.x / B.ext[2], x = y / B.ext[1];
    y -= x*B.ext[1];
    const int dz = blockDim.x % B.ext[2], dy0 = blockDim.x / B.ext[2], dx = dy0 / B.ext[1], dy = dy0 - dx*B.ext[1];
    for (int c = threadIdx.x; c < npts; c += blockDim.x) {
        const unsigned long long v = brick[c];
        if (v != 0ull)
            atomicAdd((unsigned long long*) pme.gridFixed + ((size_t) B.wrap(0, x, pme.nx)*pme.ny + B.wrap(1, y, pme.ny))*pme.nz + B.wrap(2, z, pme.nz), v);
        z += dz; y += dy; x += dx;
        if (z >= B.ext[2]) { z -= B.ext[2]; y++; }
        if (y >= B.ext[1]) { y -= B.ext[1]; x++; }
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

// allows the brick spread all the dynamic shared memory a CTA can opt in to (maxSmem bytes with their static shared memory)
// on the current device; each launch asks for what it uses
void pme_brick_setup(int maxSmem) {
    cudaFuncAttributes fa;
    CUDA_CHECK(cudaFuncGetAttributes(&fa, k_pme_spread_brick));
    CUDA_CHECK(cudaFuncSetAttribute(k_pme_spread_brick, cudaFuncAttributeMaxDynamicSharedMemorySize, maxSmem - (int) fa.sharedSizeBytes));
}

void launch_pme_spread(const NbDev& nb, const PmeDev& pme, const CommDev& cd, cudaStream_t s, bool zeroGrid) {
    if (zeroGrid) cudaMemsetAsync(pme.gridFixed, 0, sizeof(long long)*(size_t) pme.nx*pme.ny*pme.nz, s);
    if (pme.brickAtoms > 0) {
        launch_high(k_pme_spread_brick, (nb.npad + pme.brickAtoms - 1)/pme.brickAtoms, 256, sizeof(long long)*pme.brickPoints, s, nb, pme);
        return;
    }
    const int per = cd.world > 1 ? cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank] : (nb.natoms + nb.world - 1)/nb.world;
    launch_high(k_pme_spread, std::max(1, (per*8 + 127)/128), 128, 0, s, nb, pme, cd);
}

void launch_pme_gather(const NbDev& nb, const PmeDev& pme, const CommDev& cd, cudaStream_t s) {
    const int per = cd.world > 1 ? cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank] : (nb.natoms + nb.world - 1)/nb.world;
    launch_high(k_pme_gather, std::max(1, (per + 127)/128), 128, 0, s, nb, pme, cd);
}
