// fft.cu -- the bespoke grid-resident 3-D FFT for PME (sm_90a), fused with the reciprocal-space convolution.
//
// Replaces cufftExecR2C / cufftExecC2R + reciprocalConvolution + gridEvaluateEnergy of the reference CUDA
// platform (CudaKernels.cpp:826-829,1228-1255; pme.cc:390-505); numerically it restates fftpack_exec_3d +
// pme_reciprocal_convolution (ReferencePME.cpp:409-514, 793-799): unnormalised transforms in both directions,
// forward = exp(-2 pi i jk/n).
//
// Single precision spectral pipeline (typedef real, engine.h); the INPUT is the int64 fixed-point charge grid, which makes
// spreading -- and therefore every force -- independent of the order of the atomics.
//
// Three launches when two copies of a (y,z) plane fit in shared memory (grids up to ~160^2 per plane; the usual case):
//   1  k_fft_slab_fwd   one x plane per CTA: R2C along z (two real rows packed into one complex line), then along y
//   2  k_fft_x_conv     16 (ky,kz) lines per CTA: forward along x, multiply by the influence function, accumulate the
//                       reciprocal energy, inverse along x -- the k-space grid never leaves shared memory between the three
//   3  k_fft_slab_inv   one x plane per CTA: inverse along y, C2R along z
// otherwise five line-batched passes (k_fft_z_fwd, k_fft_y, k_fft_x_conv, k_fft_y, k_fft_z_inv).
//
// Multi-GPU (CommDev::world > 1): x planes are dealt to the ranks in contiguous slabs, (ky,kz) lines in contiguous chunks.
// The two transposes of a slab-decomposed 3-D FFT are the STORES of kernels 1 and 2: k_fft_slab_fwd writes every
// transformed plane straight into the line owners' buffers over NVLink, k_fft_x_conv writes its lines back into the slab
// owners' buffers, k_fft_slab_inv writes the potential plane into everybody's grid; each publishes one flag per stage
// (CH_FWD, CH_INV, CH_POT) and the consumer kernel spins on it.  k_fft_slab_fwd also sums the charge-grid contributions
// that the other ranks pushed (k_grid_push, CH_GRID) while it loads its plane.
//
// 1-D transforms are Stockham autosort, mixed radix 2..16 (any n whose prime factors are <= 13), out of place between two
// shared-memory buffers, twiddles staged in shared memory; radix 2/4 butterflies are multiplication free, odd radices use
// the conjugate-pair form.
#include "engine.h"
#include <algorithm>
#include <math.h>
#include <stdlib.h>


#define FFT_THREADS 512
#define TID (threadIdx.y*blockDim.x + threadIdx.x)
#define NTHR (blockDim.x*blockDim.y)
__device__ __forceinline__ real2 make_real2(real x, real y) { real2 r; r.x = x; r.y = y; return r; }

// One Stockham stage of radix R over `nlines` contiguous lines of length n (line l at base + l*n), one BUTTERFLY per
// thread: R inputs are read once into registers, multiplied by the stage twiddles, combined by a generic radix-R DFT
// (R*R complex MACs against the R-th roots of unity, taken from the twiddle table in shared memory) and written to their
// autosort positions.  Shared-memory traffic is 2 accesses per point per stage.  (A one-OUTPUT-per-thread variant was
// tried in round 1: R-fold redundant operand reads made the transform shared-memory-bandwidth bound, 62 us at 56^3.)
// Division of a small non-negative int by a runtime divisor as one multiply-high: exact for x < 2^32/d (all index ranges
// here are < 2^20 and d <= 4096).  The divisions by nb, Ns, nz, nzc were ~50 of the ~100 instructions per butterfly.
struct FastDiv {
    unsigned int m; int d;
    __device__ __forceinline__ explicit FastDiv(int dd) : m(dd > 1 ? 0xffffffffu/(unsigned int) dd + 1u : 0u), d(dd) {}
    __device__ __forceinline__ int div(int x) const { return d > 1 ? (int) __umulhi((unsigned int) x, m) : x; }
};

template <int R>
__device__ __forceinline__ void fft_stage(const real2* __restrict__ in, real2* __restrict__ out, int n, int nlines,
                                          int Ns, const real2* __restrict__ tw, bool inverse) {
    const int nb = n/R;                 // butterflies per line
    const int twStep = n/(Ns*R);
    const int total = nlines*nb;
    const real sgn = inverse ? (real) -1 : (real) 1;
    const FastDiv divNb(nb), divNs(Ns);
    for (int w = TID; w < total; w += NTHR) {
        const int line = divNb.div(w);
        const int j = w - line*nb;
        const int jq = divNs.div(j);
        const int k = j - jq*Ns;
        const real2* src = in + line*n + j;
        real2 v[R];
#pragma unroll
        for (int t = 0; t < R; t++) v[t] = src[t*nb];
        if (k > 0) {
            int idx = 0;
#pragma unroll
            for (int t = 1; t < R; t++) {
                idx += k*twStep;                     // t*k*twStep < n
                real2 wv = tw[idx];
                wv.y *= sgn;
                const real2 x = v[t];
                v[t] = make_real2(x.x*wv.x - x.y*wv.y, x.x*wv.y + x.y*wv.x);
            }
        }
        real2* dst = out + line*n + jq*Ns*R + k;
        if (R == 2) {
            dst[0] = make_real2(v[0].x + v[R-1].x, v[0].y + v[R-1].y);
            dst[Ns] = make_real2(v[0].x - v[R-1].x, v[0].y - v[R-1].y);
        }
        else if (R == 4) {
            // radix-4 with trivial roots (-i forward, +i inverse): 16 adds, no multiplications
            const real2 a = make_real2(v[0].x + v[R/2].x, v[0].y + v[R/2].y), b = make_real2(v[0].x - v[R/2].x, v[0].y - v[R/2].y);
            const real2 c = make_real2(v[1].x + v[R-1].x, v[1].y + v[R-1].y), d = make_real2(v[1].x - v[R-1].x, v[1].y - v[R-1].y);
            const real2 id = make_real2(sgn*d.y, -sgn*d.x);         // (-i forward / +i inverse) * d
            dst[0] = make_real2(a.x + c.x, a.y + c.y);
            dst[Ns] = make_real2(b.x + id.x, b.y + id.y);
            dst[2*Ns] = make_real2(a.x - c.x, a.y - c.y);
            dst[3*Ns] = make_real2(b.x - id.x, b.y - id.y);
        }
        else if (R & 1) {
            // odd radix, conjugate-pair form: with s_t = x_t + x_{R-t}, d_t = x_t - x_{R-t} (t = 1..h, h = (R-1)/2)
            //   X_q = x_0 + sum_t s_t cos(2 pi q t/R) -+ i sum_t d_t sin(2 pi q t/R),  X_{R-q} = conj-partner
            // i.e. h*h real-coefficient MAC pairs instead of (R-1)^2 complex MACs (radix 7: 36 FMA instead of 168).
            constexpr int H = (R - 1)/2;
            real2 sm[H > 0 ? H : 1], df[H > 0 ? H : 1];
            real2 x0 = v[0];
            real2 sum0 = x0;
#pragma unroll
            for (int t = 1; t <= H; t++) {
                sm[t-1] = make_real2(v[t].x + v[R-t].x, v[t].y + v[R-t].y);
                df[t-1] = make_real2(v[t].x - v[R-t].x, v[t].y - v[R-t].y);
                sum0.x += sm[t-1].x; sum0.y += sm[t-1].y;
            }
            dst[0] = sum0;
#pragma unroll
            for (int q = 1; q <= H; q++) {
                real2 A = x0, B = make_real2(0, 0);
#pragma unroll
                for (int t = 1; t <= H; t++) {
                    const real2 r = tw[((q*t) % R)*nb];      // (cos, -sin) of 2 pi (q t mod R)/R: warp-uniform broadcast
                    A.x += sm[t-1].x*r.x; A.y += sm[t-1].y*r.x;
                    B.x += df[t-1].x*r.y; B.y += df[t-1].y*r.y;
                }
                // forward: X_q = A + i*(B with r.y = -sin) -> A - i*sum d sin ; the inverse flips the sign of the sine part
                const real2 iB = make_real2(-sgn*B.y, sgn*B.x);                  // i*B (forward) / -i*B (inverse)
                dst[q*Ns] = make_real2(A.x + iB.x, A.y + iB.y);
                dst[(R-q)*Ns] = make_real2(A.x - iB.x, A.y - iB.y);
            }
        }
        else {
            // other even radices (6, 8, 10, ...: the planner avoids them): generic, output loop ROLLED, roots re-read from
            // shared memory as warp-uniform broadcasts
#pragma unroll 1
            for (int q = 0; q < R; q++) {
                real2 acc = v[0];
                int idx = 0;
                const int step = q*nb;
#pragma unroll
                for (int t = 1; t < R; t++) {
                    idx += step;
                    if (idx >= n) idx -= n;
                    real2 r = tw[idx];
                    r.y *= sgn;
                    acc.x += v[t].x*r.x - v[t].y*r.y;
                    acc.y += v[t].x*r.y + v[t].y*r.x;
                }
                dst[q*Ns] = acc;
            }
        }
    }
}

// full 1-D transform of `nlines` contiguous lines; returns the buffer holding the result. Block-wide.
__device__ real2* fft_lines(real2* a, real2* b, const FftPlanDev& plan, int nlines, const unsigned int* tab, const real2* tw, bool inverse) {
    (void) tab;
    int Ns = 1;
    real2* in = a;
    real2* out = b;
    for (int s = 0; s < plan.nstages; s++) {
        const int R = plan.radix[s];
        switch (R) {
            case 2: fft_stage<2>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 3: fft_stage<3>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 4: fft_stage<4>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 5: fft_stage<5>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 6: fft_stage<6>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 7: fft_stage<7>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 8: fft_stage<8>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 9: fft_stage<9>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 10: fft_stage<10>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 11: fft_stage<11>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 12: fft_stage<12>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 13: fft_stage<13>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 14: fft_stage<14>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 15: fft_stage<15>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            case 16: fft_stage<16>(in, out, plan.n, nlines, Ns, tw, inverse); break;
            default: break;
        }
        __syncthreads();
        Ns *= R;
        real2* t = in; in = out; out = t;
    }
    return in;
}

// factorisation into radices <= 16 minimising sum(R + 4): R complex MACs per point per generic stage plus a
// synchronisation cost per stage (exhaustive search, n is small)
static int best_cost(int n, int* radix, int depth) {
    if (n == 1) return 0;
    if (depth >= B200MD_MAX_FFT_STAGES) return 1 << 28;
    int best = 1 << 28, sub[B200MD_MAX_FFT_STAGES];
    for (int r = 2; r <= B200MD_MAX_RADIX && r <= n; r++) {
        if (n % r) continue;
        // radix 2 / 4: multiplication-free butterflies; odd radices: conjugate-pair form (~r/2 MACs per point); other even
        // radices fall back to the generic r MACs per point and are avoided
        const int stageCost = (r == 2 ? 2 : (r == 4 ? 3 : ((r & 1) ? (r+1)/2 + 1 : 2*r))) + 3;
        int c = stageCost + best_cost(n/r, sub, depth+1);
        if (c < best) {
            best = c;
            radix[0] = r;
            for (int k = 0; k + depth + 1 < B200MD_MAX_FFT_STAGES && k < B200MD_MAX_FFT_STAGES-1; k++) radix[k+1] = sub[k];
        }
    }
    return best;
}

bool fft_make_radices(int n, int* radix, int* nstages) {
    int r[B200MD_MAX_FFT_STAGES+1] = {0};
    if (n < 1) return false;
    if (best_cost(n, r, 0) >= (1 << 28)) return false;
    int ns = 0, rem = n;
    while (rem > 1 && ns < B200MD_MAX_FFT_STAGES) { radix[ns] = r[ns]; rem /= r[ns]; ns++; }
    if (rem != 1) return false;
    // larger radices first: the early stages have the poorest write locality, keep them few
    for (int a = 0; a < ns; a++) for (int b = a+1; b < ns; b++) if (radix[b] > radix[a]) { int t = radix[a]; radix[a] = radix[b]; radix[b] = t; }
    *nstages = ns;
    return true;
}

#define ZROWS 16          // real rows per CTA in the z passes (8 packed complex lines)
#define LINE_BATCH 16     // lines per CTA in the y and x passes

size_t fft_plane_smem_bytes(int ny, int nz) {       // kept for the engine's capacity check: largest per-CTA need
    size_t z = (2*(size_t) (ZROWS/2)*nz + 3*nz)*sizeof(real2);
    size_t y = (2*(size_t) LINE_BATCH*ny + 3*ny)*sizeof(real2);
    return z > y ? z : y;
}
size_t fft_line_smem_bytes(int nx) { return (2*(size_t) LINE_BATCH*nx + 3*nx)*sizeof(real2); }

// twiddles (n real2) followed by the per-stage position tables (8*n uint32 = 2n real2 of space)
__device__ __forceinline__ unsigned int* stage_twiddles(real2* tws, const FftPlanDev& plan) {
    for (int i = TID; i < plan.n; i += NTHR) tws[i] = plan.tw[i];
    unsigned int* tab = (unsigned int*) (tws + plan.n);
    return tab;
}

// ---- 1: forward z, real to complex, two rows per complex line ----
__global__ void __launch_bounds__(FFT_THREADS) k_fft_z_fwd(PmeDev pme) {
    extern __shared__ real2 smem[];
    const int nz = pme.nz, nzc = pme.nzc;
    const FastDiv divNz(nz), divNzc(nzc);
    const int nrowsTotal = pme.nx*pme.ny;
    const int row0 = blockIdx.x*ZROWS;
    const int nrows = min(ZROWS, nrowsTotal - row0);
    const int np = (nrows + 1)/2;
    real2* A = smem;
    real2* B = A + (ZROWS/2)*nz;
    real2* tws = B + (ZROWS/2)*nz;
    const unsigned int* tab = stage_twiddles(tws, pme.plan[2]);
    if (pme.gridFixed != nullptr) {
        const long long* base = pme.gridFixed + (size_t) row0*nz;
        for (int i = TID; i < np*nz; i += NTHR) {
            const int p = divNz.div(i), z = i - p*nz;
            const real re = fixed_to_float(base[(size_t) (2*p)*nz + z]);
            const real im = (2*p+1 < nrows) ? fixed_to_float(base[(size_t) (2*p+1)*nz + z]) : (real) 0;
            A[i] = make_real2(re, im);
        }
    }
    else {
        const real* base = pme.grid + (size_t) row0*nz;
        for (int i = TID; i < np*nz; i += NTHR) {
            const int p = divNz.div(i), z = i - p*nz;
            const real re = base[(size_t) (2*p)*nz + z];
            const real im = (2*p+1 < nrows) ? base[(size_t) (2*p+1)*nz + z] : (real) 0;
            A[i] = make_real2(re, im);
        }
    }
    __syncthreads();
    const real2* R = fft_lines(A, B, pme.plan[2], np, tab, tws, false);
    // unpack the two interleaved real transforms straight to global memory
    real2* dst = pme.cgrid + (size_t) row0*nzc;
    for (int i = TID; i < np*nzc; i += NTHR) {
        const int p = divNzc.div(i), k = i - p*nzc;
        const real2 Z = R[p*nz + k];
        real2 Zc = R[p*nz + (k == 0 ? 0 : nz - k)];
        Zc.y = -Zc.y;
        dst[(size_t) (2*p)*nzc + k] = make_real2((real) 0.5*(Z.x + Zc.x), (real) 0.5*(Z.y + Zc.y));
        if (2*p+1 < nrows) {
            const real2 d = make_real2((real) 0.5*(Z.x - Zc.x), (real) 0.5*(Z.y - Zc.y));
            dst[(size_t) (2*p+1)*nzc + k] = make_real2(d.y, -d.x);     // -i*d
        }
    }
}

// ---- 5: inverse z, complex to real ----
__global__ void __launch_bounds__(FFT_THREADS) k_fft_z_inv(PmeDev pme) {
    extern __shared__ real2 smem[];
    const int nz = pme.nz, nzc = pme.nzc;
    const FastDiv divNz(nz), divNzc(nzc);
    const int nrowsTotal = pme.nx*pme.ny;
    const int row0 = blockIdx.x*ZROWS;
    const int nrows = min(ZROWS, nrowsTotal - row0);
    const int np = (nrows + 1)/2;
    real2* A = smem;
    real2* B = A + (ZROWS/2)*nz;
    real2* tws = B + (ZROWS/2)*nz;
    const unsigned int* tab = stage_twiddles(tws, pme.plan[2]);
    const real2* src = pme.cgrid + (size_t) row0*nzc;
    // pack rows (2p, 2p+1) into one complex line using the Hermitian symmetry along z
    for (int i = TID; i < np*nz; i += NTHR) {
        const int p = divNz.div(i), k = i - p*nz;
        const int kk = (k < nzc) ? k : nz - k;
        real2 a = src[(size_t) (2*p)*nzc + kk];
        real2 b = (2*p+1 < nrows) ? src[(size_t) (2*p+1)*nzc + kk] : make_real2(0, 0);
        if (k >= nzc) { a.y = -a.y; b.y = -b.y; }
        A[i] = make_real2(a.x - b.y, a.y + b.x);       // a + i b
    }
    __syncthreads();
    const real2* Z = fft_lines(A, B, pme.plan[2], np, tab, tws, true);
    real* dst = pme.grid + (size_t) row0*nz;
    for (int i = TID; i < np*nz; i += NTHR) {
        const int p = divNz.div(i), z = i - p*nz;
        const real2 v = Z[i];
        dst[(size_t) (2*p)*nz + z] = v.x;
        if (2*p+1 < nrows) dst[(size_t) (2*p+1)*nz + z] = v.y;
    }
}

// ---- 2 / 4: along y, LINE_BATCH adjacent kz columns of one x per CTA ----
__global__ void __launch_bounds__(FFT_THREADS) k_fft_y(PmeDev pme, int inverse) {
    extern __shared__ real2 smem[];
    const int ny = pme.ny, nzc = pme.nzc;
    const int nbz = (nzc + LINE_BATCH - 1)/LINE_BATCH;
    const int x = blockIdx.x/nbz, bz = blockIdx.x - x*nbz;
    const int kz0 = bz*LINE_BATCH;
    const int nk = min(LINE_BATCH, nzc - kz0);
    real2* A = smem;
    real2* B = A + LINE_BATCH*ny;
    real2* tws = B + LINE_BATCH*ny;
    const unsigned int* tab = stage_twiddles(tws, pme.plan[1]);
    real2* base = pme.cgrid + (size_t) x*ny*nzc + kz0;
    for (int i = TID; i < ny*LINE_BATCH; i += NTHR) {
        const int y = i/LINE_BATCH, l = i - y*LINE_BATCH;
        if (l < nk) A[l*ny + y] = base[(size_t) y*nzc + l];
    }
    __syncthreads();
    const real2* R = fft_lines(A, B, pme.plan[1], nk, tab, tws, inverse != 0);
    for (int i = TID; i < ny*LINE_BATCH; i += NTHR) {
        const int y = i/LINE_BATCH, l = i - y*LINE_BATCH;
        if (l < nk) base[(size_t) y*nzc + l] = R[l*ny + y];
    }
}

// ---- 3: forward x, convolution + energy, inverse x; one batch of (ky,kz) lines per CTA ----
// mode 0: forward + convolution + inverse (PME); mode 1: forward only; mode 2: inverse only (stand-alone FFT)
template <bool ENERGY>
__global__ void __launch_bounds__(FFT_THREADS) k_fft_x_conv(PmeDev pme, double* energyOut, int mode, CommDev cd) {
    extern __shared__ real2 smem[];
    const int nx = pme.nx;
    const int plane = pme.ny*pme.nzc;
    real2* A = smem;
    real2* B = A + LINE_BATCH*nx;
    real2* tws = B + LINE_BATCH*nx;
    const unsigned int* tab = stage_twiddles(tws, pme.plan[0]);
    const bool multi = cd.world > 1;
    const unsigned long long E = multi ? *cd.epoch + 1ull : 0ull;
    // multi-GPU: this rank's chunk of lines [mlo, mlo + mcount) arrives in its line buffer, layout [x][mcount]
    const int mlo = multi ? cd.rank*cd.lineChunk : 0;
    const int mcount = multi ? max(0, min(cd.lineChunk, plane - mlo)) : plane;
    const real2* src = multi ? (const real2*) (cd.peer[cd.rank] + cd.offLineBuf) : pme.cgrid;
    if (multi) comm_wait(cd, CH_FWD, E);
    const int m0 = blockIdx.x*LINE_BATCH;
    const int nl = min(LINE_BATCH, mcount - m0);
    for (int i = TID; i < nx*LINE_BATCH; i += NTHR) {
        const int x = i/LINE_BATCH, l = i - x*LINE_BATCH;
        if (l < nl) A[l*nx + x] = src[(size_t) x*mcount + m0 + l];
    }
    __syncthreads();
    real2* R = A;
    real2* other = B;
    if (mode != 2) {
        R = fft_lines(A, B, pme.plan[0], max(nl, 0), tab, tws, false);
        other = (R == A) ? B : A;
    }
    if (mode == 0) {
        double esum = 0.0;
        for (int i = TID; i < nx*LINE_BATCH; i += NTHR) {
            const int x = i/LINE_BATCH, l = i - x*LINE_BATCH;
            if (l < nl) {
                const int m = mlo + m0 + l;
                const real et = pme.eterm[(size_t) x*plane + m];
                const real2 v = R[l*nx + x];
                if (ENERGY) {
                    const int kz = m % pme.nzc;
                    const double wgt = (kz == 0 || (2*kz == pme.nz)) ? 1.0 : 2.0;    // Hermitian mirror counted here
                    esum += wgt*et*(v.x*v.x + v.y*v.y);
                }
                R[l*nx + x] = make_real2(v.x*et, v.y*et);
            }
        }
        if (ENERGY) {
            __shared__ double red[32];
            for (int off = 16; off > 0; off >>= 1) esum += __shfl_xor_sync(0xffffffffu, esum, off);
            if ((TID & 31) == 0) red[TID >> 5] = esum;
            __syncthreads();
            if (TID == 0) {
                double tot = 0.0;
                for (int w = 0; w < (NTHR + 31)/32; w++) tot += red[w];
                atomicAdd(energyOut, 0.5*tot);
            }
        }
        __syncthreads();
    }
    if (mode != 1)
        R = fft_lines(R, other, pme.plan[0], max(nl, 0), tab, tws, true);
    if (multi) {
        // second transpose: every x plane goes back to the rank that owns its slab, layout [x - xLo][plane]
        for (int i = TID; i < nx*LINE_BATCH; i += NTHR) {
            const int x = i/LINE_BATCH, l = i - x*LINE_BATCH;
            if (l < nl) {
                int q = 0;
#pragma unroll
                for (int k = 1; k < B200MD_MAX_RANKS; k++) q += (k < cd.world && x >= cd.xLo[k]) ? 1 : 0;
                ((real2*) (cd.peer[q] + cd.offPlaneBuf))[(size_t) (x - cd.xLo[q])*plane + mlo + m0 + l] = R[l*nx + x];
            }
        }
        comm_signal(cd, CH_INV, E, gridDim.x);
        return;
    }
    for (int i = TID; i < nx*LINE_BATCH; i += NTHR) {
        const int x = i/LINE_BATCH, l = i - x*LINE_BATCH;
        if (l < nl) pme.cgrid[(size_t) x*plane + m0 + l] = R[l*nx + x];
    }
}

static void set_smem(const void* f, size_t bytes) {
    if (bytes > 48*1024) cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) bytes);
}

// ---- slab kernels: one x-slab per CTA, the whole (y,z) plane lives in shared memory, z and y passes fused ----
// Used whenever 2 plane buffers fit in shared memory (ny*nzc <= ~6900 points, i.e. grids up to ~112^2 per slab); then
// forward + convolution + inverse is THREE launches (slab fwd, x lines + convolution, slab inv), which matters because
// at 56^3 every launch boundary costs more than the arithmetic of a whole pass.
struct SlabSmem { real2 *A, *B, *twz, *twy; unsigned int *tabz, *taby; };

__device__ __forceinline__ SlabSmem slab_setup(real2* smem, const PmeDev& pme, size_t elems) {
    SlabSmem S;
    S.A = smem; S.B = smem + elems;
    S.twz = S.B + elems; S.twy = S.twz + pme.nz;
    S.tabz = (unsigned int*) (S.twy + pme.ny);
    S.taby = S.tabz + 8*pme.nz;
    for (int i = TID; i < pme.nz; i += NTHR) S.twz[i] = pme.plan[2].tw[i];
    for (int i = TID; i < pme.ny; i += NTHR) S.twy[i] = pme.plan[1].tw[i];
    return S;
}

static size_t slab_elems(const PmeDev& p) {
    const size_t np = (p.ny + 1)/2;
    size_t e = (size_t) p.ny*p.nzc;
    if (np*p.nz > e) e = np*p.nz;
    return e;
}
static size_t slab_smem_bytes(const PmeDev& p) {
    return 2*slab_elems(p)*sizeof(real2) + (size_t) (p.nz + p.ny)*sizeof(real2) + (size_t) 8*(p.nz + p.ny)*sizeof(unsigned int);
}

__global__ void __launch_bounds__(FFT_THREADS) k_fft_slab_fwd(PmeDev pme, size_t elems, CommDev cd) {
    extern __shared__ real2 smem[];
    const int ny = pme.ny, nz = pme.nz, nzc = pme.nzc;
    const FastDiv divNz(nz), divNzc(nzc);
    const int np = (ny + 1)/2;
    SlabSmem S = slab_setup(smem, pme, elems);
    const bool multi = cd.world > 1;
    const unsigned long long E = multi ? *cd.epoch + 1ull : 0ull;
    const int x = (multi ? cd.xLo[cd.rank] : 0) + blockIdx.x;
    if (multi) {
        // the plane = this rank's own spread + what the other ranks pushed into the inboxes (exact int64 sums)
        comm_wait(cd, CH_GRID, E);
        const size_t planeCells = (size_t) ny*nz;
        const long long* own = pme.gridFixed + (size_t) x*planeCells;
        const long long* inbox = (const long long*) (cd.peer[cd.rank] + cd.offGridInbox) + (size_t) (x - cd.xLo[cd.rank])*planeCells;
        const size_t inboxStride = (size_t) cd.maxPlanes*planeCells;
        for (int i = TID; i < np*nz; i += NTHR) {
            const int p = divNz.div(i), z = i - p*nz;
            long long a = own[(size_t) (2*p)*nz + z], b = (2*p+1 < ny) ? own[(size_t) (2*p+1)*nz + z] : 0ll;
            for (int q = 0; q < cd.world; q++) if (q != cd.rank) {
                const long long* iq = inbox + (size_t) q*inboxStride;
                a += iq[(size_t) (2*p)*nz + z];
                if (2*p+1 < ny) b += iq[(size_t) (2*p+1)*nz + z];
            }
            S.A[i] = make_real2(fixed_to_float(a), fixed_to_float(b));
        }
    }
    else if (pme.gridFixed != nullptr) {
        long long* base = pme.gridFixed + (size_t) x*ny*nz;
        for (int i = TID; i < np*nz; i += NTHR) {
            const int p = divNz.div(i), z = i - p*nz;
            const real re = fixed_to_float(base[(size_t) (2*p)*nz + z]);
            const real im = (2*p+1 < ny) ? fixed_to_float(base[(size_t) (2*p+1)*nz + z]) : (real) 0;
            S.A[i] = make_real2(re, im);
        }
    }
    else {
        const real* base = pme.grid + (size_t) x*ny*nz;
        for (int i = TID; i < np*nz; i += NTHR) {
            const int p = divNz.div(i), z = i - p*nz;
            S.A[i] = make_real2(base[(size_t) (2*p)*nz + z], (2*p+1 < ny) ? base[(size_t) (2*p+1)*nz + z] : 0.0);
        }
    }
    __syncthreads();
    const real2* R = fft_lines(S.A, S.B, pme.plan[2], np, S.tabz, S.twz, false);
    real2* O = (R == S.A) ? S.B : S.A;
    // unpack the two interleaved real transforms, transposed to [kz][y] so that the y lines are contiguous
    for (int i = TID; i < np*nzc; i += NTHR) {
        const int p = divNzc.div(i), k = i - p*nzc;
        const real2 Z = R[p*nz + k];
        real2 Zc = R[p*nz + (k == 0 ? 0 : nz - k)];
        Zc.y = -Zc.y;
        O[k*ny + 2*p] = make_real2((real) 0.5*(Z.x + Zc.x), (real) 0.5*(Z.y + Zc.y));
        if (2*p+1 < ny) {
            const real2 d = make_real2((real) 0.5*(Z.x - Zc.x), (real) 0.5*(Z.y - Zc.y));
            O[k*ny + 2*p+1] = make_real2(d.y, -d.x);
        }
    }
    __syncthreads();
    real2* other = (O == S.A) ? S.B : S.A;
    const real2* Y = fft_lines(O, other, pme.plan[1], nzc, S.taby, S.twy, false);
    if (multi) {
        // first transpose: line m = y*nzc + k of this plane goes to the rank that owns the line, layout [x][its line count]
        const int plane = ny*nzc;
        const FastDiv divChunk(cd.lineChunk);
        for (int i = TID; i < plane; i += NTHR) {
            const int y = divNzc.div(i), k = i - y*nzc;
            const int q = divChunk.div(i);
            const int mq = i - q*cd.lineChunk;
            const int cnt = min(cd.lineChunk, plane - q*cd.lineChunk);
            ((real2*) (cd.peer[q] + cd.offLineBuf))[(size_t) x*cnt + mq] = Y[k*ny + y];
        }
        comm_signal(cd, CH_FWD, E, gridDim.x);
        return;
    }
    real2* dst = pme.cgrid + (size_t) x*ny*nzc;
    for (int i = TID; i < ny*nzc; i += NTHR) {
        const int y = divNzc.div(i), k = i - y*nzc;
        dst[i] = Y[k*ny + y];
    }
}

__global__ void __launch_bounds__(FFT_THREADS) k_fft_slab_inv(PmeDev pme, size_t elems, CommDev cd) {
    extern __shared__ real2 smem[];
    const int ny = pme.ny, nz = pme.nz, nzc = pme.nzc;
    const FastDiv divNz(nz), divNzc(nzc);
    const int np = (ny + 1)/2;
    SlabSmem S = slab_setup(smem, pme, elems);
    const bool multi = cd.world > 1;
    const unsigned long long E = multi ? *cd.epoch + 1ull : 0ull;
    const int x = (multi ? cd.xLo[cd.rank] : 0) + blockIdx.x;
    if (multi) comm_wait(cd, CH_INV, E);
    const real2* src = multi ? (const real2*) (cd.peer[cd.rank] + cd.offPlaneBuf) + (size_t) (x - cd.xLo[cd.rank])*ny*nzc
                             : pme.cgrid + (size_t) x*ny*nzc;
    for (int i = TID; i < ny*nzc; i += NTHR) {
        const int y = divNzc.div(i), k = i - y*nzc;
        S.A[k*ny + y] = src[i];
    }
    __syncthreads();
    const real2* Y = fft_lines(S.A, S.B, pme.plan[1], nzc, S.taby, S.twy, true);
    real2* O = (Y == S.A) ? S.B : S.A;
    // pack rows (2p, 2p+1) into one complex line using the Hermitian symmetry along z
    for (int i = TID; i < np*nz; i += NTHR) {
        const int p = divNz.div(i), k = i - p*nz;
        const int kk = (k < nzc) ? k : nz - k;
        real2 a = Y[kk*ny + 2*p];
        real2 b = (2*p+1 < ny) ? Y[kk*ny + 2*p+1] : make_real2(0, 0);
        if (k >= nzc) { a.y = -a.y; b.y = -b.y; }
        O[i] = make_real2(a.x - b.y, a.y + b.x);
    }
    __syncthreads();
    real2* other = (O == S.A) ? S.B : S.A;
    const real2* Z = fft_lines(O, other, pme.plan[2], np, S.tabz, S.twz, true);
    if (multi) {
        // the potential plane goes into EVERY rank's grid (each rank interpolates the forces of its own atoms, wherever they are)
        for (int k = 0; k < cd.world; k++) {
            const int q = (cd.rank + k) % cd.world;              // own copy first, then the peers in staggered order
            real* dq = (real*) (cd.peer[q] + cd.offGrid) + (size_t) x*ny*nz;
            for (int i = TID; i < np*nz; i += NTHR) {
                const int p = divNz.div(i), z = i - p*nz;
                const real2 v = Z[i];
                dq[(size_t) (2*p)*nz + z] = v.x;
                if (2*p+1 < ny) dq[(size_t) (2*p+1)*nz + z] = v.y;
            }
        }
        comm_signal(cd, CH_POT, E, gridDim.x);
        return;
    }
    real* dst = pme.grid + (size_t) x*ny*nz;
    for (int i = TID; i < np*nz; i += NTHR) {
        const int p = divNz.div(i), z = i - p*nz;
        const real2 v = Z[i];
        dst[(size_t) (2*p)*nz + z] = v.x;
        if (2*p+1 < ny) dst[(size_t) (2*p+1)*nz + z] = v.y;
    }
}

// Threads per CTA.  The kernels are compiled for up to 512 threads at 128 registers, i.e. a 512-thread CTA owns a whole SM's
// register file.  A (y,z) plane keeps 512 threads busy only in its load / store phases (a radix-11 stage of an 88-point
// line has 8 butterflies per line), a batch of 16 x lines even less.  On one GPU (besideTiles) the chain runs beside the
// tile kernel, whose four CTAs per SM hold the whole register file: a 128-thread CTA (about 13,000 registers) fits the
// slot that one retiring tile CTA hands back, a 512-thread CTA would wait for an SM to drain.  With an SM partition
// (multi-GPU) smaller CTAs let 2-4 of them share one of the few SMs the chain has.  Every butterfly is computed the same
// way whichever thread takes it, so the shape does not change a bit of the result.
// B200MD_FFT_THREADS / B200MD_FFTX_THREADS override (slab kernels / x-line kernel).
static int g_fft_compact = 0;            // fft_set_compact(): the chain runs on a reserved subset of the SMs; 2 = fewer SMs than planes per rank
void fft_set_compact(int on) { g_fft_compact = on; }
static int fft_threads(bool besideTiles) {
    static const int env = getenv("B200MD_FFT_THREADS") ? std::min(FFT_THREADS, std::max(64, atoi(getenv("B200MD_FFT_THREADS")))) : 0;
    if (env) return env;
    if (besideTiles) return 128;
    return g_fft_compact == 2 ? 256 : FFT_THREADS;       // a plane per SM when there is one: 512 threads finish it in ~2/3 of the time of 256
}
static int fftx_threads(bool besideTiles) {
    static const int env = getenv("B200MD_FFTX_THREADS") ? std::min(FFT_THREADS, std::max(64, atoi(getenv("B200MD_FFTX_THREADS")))) : 0;
    return env ? env : (g_fft_compact ? 128 : fft_threads(besideTiles));
}

struct FftLaunch {
    size_t zs, ys, xs, ss, selems;
    int zb, yb, xb;
    dim3 zt, yt, xt, st;
    bool slab;
    FftLaunch(const PmeDev& p, bool besideTiles = false) {
        int dev = 0, maxSmem = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&maxSmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
        ss = slab_smem_bytes(p);
        selems = slab_elems(p);
        const int nmax = p.ny > p.nz ? p.ny : p.nz;
        slab = ss <= (size_t) maxSmem && nmax <= 1024 && getenv("B200MD_FFT_NOSLAB") == nullptr;
        if (slab) {
            st = dim3(fft_threads(besideTiles));
            set_smem((const void*) k_fft_slab_fwd, ss);
            set_smem((const void*) k_fft_slab_inv, ss);
        }
        zs = (2*(size_t) (ZROWS/2)*p.nz + 3*p.nz)*sizeof(real2);
        ys = (2*(size_t) LINE_BATCH*p.ny + 3*p.ny)*sizeof(real2);
        xs = (2*(size_t) LINE_BATCH*p.nx + 3*p.nx)*sizeof(real2);
        zt = yt = dim3(fft_threads(besideTiles)); xt = dim3(fftx_threads(besideTiles));
        zb = (p.nx*p.ny + ZROWS - 1)/ZROWS;
        yb = p.nx*((p.nzc + LINE_BATCH - 1)/LINE_BATCH);
        xb = (p.ny*p.nzc + LINE_BATCH - 1)/LINE_BATCH;
        set_smem((const void*) k_fft_z_fwd, zs);
        set_smem((const void*) k_fft_z_inv, zs);
        set_smem((const void*) k_fft_y, ys);
        set_smem((const void*) k_fft_x_conv<true>, xs);
        set_smem((const void*) k_fft_x_conv<false>, xs);
    }
};

static const CommDev g_single = [] { CommDev c{}; c.world = 1; return c; }();
static void fwd_zy(const FftLaunch& L, const PmeDev& pme, cudaStream_t s) {
    if (L.slab) launch_high(k_fft_slab_fwd, pme.nx, L.st, L.ss, s, pme, L.selems, g_single);
    else {
        launch_high(k_fft_z_fwd, L.zb, L.zt, L.zs, s, pme);
        launch_high(k_fft_y, L.yb, L.yt, L.ys, s, pme, 0);
    }
}
static void inv_yz(const FftLaunch& L, const PmeDev& pme, cudaStream_t s) {
    if (L.slab) launch_high(k_fft_slab_inv, pme.nx, L.st, L.ss, s, pme, L.selems, g_single);
    else {
        launch_high(k_fft_y, L.yb, L.yt, L.ys, s, pme, 1);
        launch_high(k_fft_z_inv, L.zb, L.zt, L.zs, s, pme);
    }
}

int pme_fft_launch_count(const PmeDev& pme) { FftLaunch L(pme); return L.slab ? 3 : 5; }

bool fft_slab_path(const PmeDev& pme) { FftLaunch L(pme); return L.slab; }

size_t fft_cta_smem_bytes(const PmeDev& pme) {
    FftLaunch L(pme, true);
    const void* kernels[] = {(const void*) k_fft_slab_fwd, (const void*) k_fft_slab_inv, (const void*) k_fft_x_conv<true>,
                             (const void*) k_fft_x_conv<false>, (const void*) k_fft_z_fwd, (const void*) k_fft_z_inv, (const void*) k_fft_y};
    size_t stat = 0;
    for (const void* k : kernels) {
        cudaFuncAttributes fa;
        CUDA_CHECK(cudaFuncGetAttributes(&fa, k));
        stat = std::max(stat, fa.sharedSizeBytes);
    }
    const size_t dyn = L.slab ? std::max(L.ss, L.xs) : std::max(L.zs, std::max(L.ys, L.xs));
    return dyn + stat;
}

void launch_pme_fft_conv(const NbDev& nb, const PmeDev& pme, const CommDev& cd, bool energy, bool besideTiles, cudaStream_t s) {
    FftLaunch L(pme, besideTiles);
    if (cd.world > 1) {
        // slab-decomposed over the ranks (the slab path is a precondition, checked when the communicator is set up)
        const int planes = cd.xLo[cd.rank + 1] - cd.xLo[cd.rank];
        const int plane = pme.ny*pme.nzc;
        const int mcount = std::max(0, std::min(cd.lineChunk, plane - cd.rank*cd.lineChunk));
        const int xb = std::max(1, (mcount + LINE_BATCH - 1)/LINE_BATCH);
        launch_high(k_fft_slab_fwd, std::max(1, planes), L.st, L.ss, s, pme, L.selems, cd);
        launch_high(energy ? k_fft_x_conv<true> : k_fft_x_conv<false>, xb, L.xt, L.xs, s, pme, nb.energy + EN_RECIP, 0, cd);
        launch_high(k_fft_slab_inv, std::max(1, planes), L.st, L.ss, s, pme, L.selems, cd);
        return;
    }
    fwd_zy(L, pme, s);
    launch_high(energy ? k_fft_x_conv<true> : k_fft_x_conv<false>, L.xb, L.xt, L.xs, s, pme, nb.energy + EN_RECIP, 0, g_single);
    inv_yz(L, pme, s);
}

void launch_fft3d_r2c(const PmeDev& pme, cudaStream_t s) {
    FftLaunch L(pme);
    fwd_zy(L, pme, s);
    launch_high(k_fft_x_conv<false>, L.xb, L.xt, L.xs, s, pme, (double*) nullptr, 1, g_single);
}

void launch_fft3d_c2r(const PmeDev& pme, cudaStream_t s) {
    FftLaunch L(pme);
    launch_high(k_fft_x_conv<false>, L.xb, L.xt, L.xs, s, pme, (double*) nullptr, 2, g_single);
    inv_yz(L, pme, s);
}
