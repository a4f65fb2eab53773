// comm.cu -- the peer-memory data plane of the multi-GPU engine (sm_90a, NVLink / NVSwitch).
//
// What the reference does here: CudaParallelKernels.cpp:110-121, 177-252 -- every device computes a share of the forces
// on ALL atoms, the host copies the partial force buffers to device 0 through pinned memory, device 0 sums and integrates
// everything, and the new positions are broadcast through the host again; reciprocal space stays on device 0
// (CudaKernels.cpp:715).  Here nothing passes through the host and no library collective is called on the step path:
// the kernels below (and k_integrate, k_pme_*, k_fft_* in their multi-rank form) store straight into the peers' windows
// over NVLink and publish one flag per stage (engine.h: CommDev, comm_wait, comm_signal).
//
//   k_force_push    partial int64 forces of the atoms this rank does not own -> the owners' inboxes (and zero them here)
//   k_integrate     (integrate.cu) owner: total = own partial + inboxes, integrate + constrain, new positions -> every rank
//   k_force_total   compute path only (energies, getState): owners total their atoms and broadcast the totals
//   k_grid_push     this rank's charge-grid contribution, slab by slab -> the slab owners' inboxes
//   k_vel_push      velocities of the owner's atoms -> every rank (before any read of the velocities from the host)
#include "engine.h"
#include <algorithm>
#include "../../include/b200md.h"

__device__ __forceinline__ long long* win_force(const CommDev& cd, int q) { return (long long*) (cd.peer[q] + cd.offForce); }
__device__ __forceinline__ long long* win_finbox(const CommDev& cd, int q, int src, int npad) { return (long long*) (cd.peer[q] + cd.offFinbox) + (size_t) src*3*npad; }

__global__ void __launch_bounds__(256) k_force_push(NbDev nb, CommDev cd) {
    const unsigned long long E = *cd.epoch + 1ull;
    const int stride = gridDim.x*blockDim.x;
    for (int a = blockIdx.x*blockDim.x + threadIdx.x; a < nb.natoms; a += stride) {
        if (a >= cd.atomLo[cd.rank] && a < cd.atomLo[cd.rank + 1]) continue;
        const int q = comm_owner_of_atom(cd, a);
        long long* in = win_finbox(cd, q, cd.rank, nb.npad);
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const size_t i = (size_t) c*nb.npad + a;
            in[i] = nb.force[i];          // unconditional: the inbox needs no zeroing between steps
            nb.force[i] = 0;
        }
    }
    comm_signal(cd, CH_FORCE, E, gridDim.x);
}

// compute path: total force of the owner's atoms = own partial + inboxes, written to every rank's force buffer
__global__ void __launch_bounds__(256) k_force_total(NbDev nb, CommDev cd) {
    const unsigned long long E = *cd.epoch + 1ull;
    comm_wait(cd, CH_FORCE, E);
    const int lo = cd.atomLo[cd.rank], hi = cd.atomLo[cd.rank + 1];
    const int stride = gridDim.x*blockDim.x;
    for (int a = lo + blockIdx.x*blockDim.x + threadIdx.x; a < hi; a += stride) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
            const size_t i = (size_t) c*nb.npad + a;
            long long f = nb.force[i];
            for (int q = 0; q < cd.world; q++) if (q != cd.rank) f += win_finbox(cd, cd.rank, q, nb.npad)[i];
            for (int k = 0; k < cd.world; k++) win_force(cd, (cd.rank + k) % cd.world)[i] = f;
        }
    }
    comm_signal(cd, CH_FINAL, E, gridDim.x);
}
// ... and everybody waits for everybody's totals; the exchange is complete, advance the epoch
__global__ void k_final_wait(CommDev cd, int ch) {
    const unsigned long long E = *cd.epoch + 1ull;
    comm_wait(cd, ch, E);
    if (threadIdx.x == 0) *cd.epoch = E;
}

__global__ void __launch_bounds__(256) k_vel_push(NbDev nb, CommDev cd) {
    const unsigned long long E = *cd.epoch + 1ull;
    const int lo = cd.atomLo[cd.rank], hi = cd.atomLo[cd.rank + 1];
    const int stride = gridDim.x*blockDim.x;
    for (int a = lo + blockIdx.x*blockDim.x + threadIdx.x; a < hi; a += stride) {
        const float4 v = nb.velm[a];
        for (int k = 1; k < cd.world; k++) ((float4*) (cd.peer[(cd.rank + k) % cd.world] + cd.offVelm))[a] = v;
    }
    comm_signal(cd, CH_VEL, E, gridDim.x);
}

// wait until the peers' position stores of the last step have landed here (host reads of the replicated state)
__global__ void k_pos_wait(CommDev cd) {
    comm_wait(cd, CH_POS, *cd.posNeed);
}

// this rank's contribution to the charge grid (int64 fixed point, from the atoms it owns), slab by slab into the inbox
// that the slab's owner keeps for this rank.  blockIdx.y = peer (skipping this rank), 16-byte loads and stores.
__global__ void __launch_bounds__(256) k_grid_push(PmeDev pme, CommDev cd) {
    const unsigned long long E = *cd.epoch + 1ull;
    const size_t planeCells = (size_t) pme.ny*pme.nz;
    const size_t inboxStride = (size_t) cd.maxPlanes*planeCells;
    const int q = (cd.rank + 1 + (int) blockIdx.y) % cd.world;            // staggered: the ranks do not all start with peer 0
    const size_t begin = (size_t) cd.xLo[q]*planeCells, cells = (size_t) (cd.xLo[q+1] - cd.xLo[q])*planeCells;
    const long long* src = pme.gridFixed + begin;
    long long* dst = (long long*) (cd.peer[q] + cd.offGridInbox) + (size_t) cd.rank*inboxStride;
    const size_t stride = (size_t) gridDim.x*blockDim.x;
    if ((begin & 1) == 0 && ((((size_t) cd.rank*inboxStride) & 1) == 0)) {      // 16-byte aligned on both sides
        const size_t pairs = cells >> 1;
        const ulonglong2* s2 = (const ulonglong2*) src;
        ulonglong2* d2 = (ulonglong2*) dst;
        for (size_t i = (size_t) blockIdx.x*blockDim.x + threadIdx.x; i < pairs; i += stride) d2[i] = s2[i];
        if ((cells & 1) && blockIdx.x == 0 && threadIdx.x == 0) dst[cells-1] = src[cells-1];
    }
    else
        for (size_t i = (size_t) blockIdx.x*blockDim.x + threadIdx.x; i < cells; i += stride) dst[i] = src[i];
    comm_signal(cd, CH_GRID, E, gridDim.x*gridDim.y);
}

// ---- the same push with the TMA engine (cp.async.bulk), used whenever the slabs are 16-byte aligned ----
// Stores into peer memory issued by threads are bound by the number of stores an SM keeps in flight: ~6 GB/s per SM,
// i.e. 4 MB took 31 us from the 22 SMs the reciprocal-space chain has at 4 ranks (profiles/r02_multi_gpu.md).  A bulk copy
// is ONE instruction per 16 KB: a single thread per CTA streams global -> shared (cp.async.bulk + mbarrier complete_tx)
// and shared -> the peer's window (cp.async.bulk.global.shared::cta, bulk groups) through a 4-stage ring, and the copy
// engines keep the links busy whatever the SM count.  SASS: UBLKCP.
#define PUSH_CHUNK 16384
#define PUSH_STAGES 4
__device__ __forceinline__ unsigned int smem_u32(const void* p) { return (unsigned int) __cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(unsigned int bar, unsigned int parity) {
    asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}" :: "r"(bar), "r"(parity) : "memory");
}
__global__ void __launch_bounds__(32) k_grid_push_tma(PmeDev pme, CommDev cd, int chunksPerCta) {
    extern __shared__ __align__(128) unsigned char ring[];            // PUSH_STAGES x PUSH_CHUNK
    __shared__ __align__(8) unsigned long long bars[PUSH_STAGES];
    const unsigned long long E = *cd.epoch + 1ull;
    const size_t planeCells = (size_t) pme.ny*pme.nz;
    const size_t inboxStride = (size_t) cd.maxPlanes*planeCells;
    const int q = (cd.rank + 1 + (int) blockIdx.y) % cd.world;            // staggered: the ranks do not all start with peer 0
    const size_t bytes = (size_t) (cd.xLo[q+1] - cd.xLo[q])*planeCells*sizeof(long long);
    const char* src = (const char*) (pme.gridFixed + (size_t) cd.xLo[q]*planeCells);
    char* dst = (char*) ((long long*) (cd.peer[q] + cd.offGridInbox) + (size_t) cd.rank*inboxStride);
    const size_t first = (size_t) blockIdx.x*chunksPerCta*PUSH_CHUNK;
    const size_t left = first < bytes ? (bytes - first + PUSH_CHUNK - 1)/PUSH_CHUNK : 0;
    const int n = (int) (left < (size_t) chunksPerCta ? left : (size_t) chunksPerCta);
    if (threadIdx.x == 0 && n > 0) {
        for (int s = 0; s < PUSH_STAGES; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bars[s])));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        auto chunk_bytes = [&](int c) { const size_t r = bytes - first - (size_t) c*PUSH_CHUNK; return (unsigned int) (r < (size_t) PUSH_CHUNK ? r : (size_t) PUSH_CHUNK); };
        auto load = [&](int c) {
            const unsigned int bar = smem_u32(&bars[c % PUSH_STAGES]), nb = chunk_bytes(c);
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(nb) : "memory");
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         :: "r"(smem_u32(ring + (size_t) (c % PUSH_STAGES)*PUSH_CHUNK)), "l"(src + first + (size_t) c*PUSH_CHUNK), "r"(nb), "r"(bar) : "memory");
        };
        const int ahead = PUSH_STAGES - 1;
        for (int c = 0; c < n && c < ahead; c++) load(c);
        for (int c = 0; c < n; c++) {
            mbar_wait(smem_u32(&bars[c % PUSH_STAGES]), (unsigned int) ((c/PUSH_STAGES) & 1));
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         :: "l"(dst + first + (size_t) c*PUSH_CHUNK), "r"(smem_u32(ring + (size_t) (c % PUSH_STAGES)*PUSH_CHUNK)), "r"(chunk_bytes(c)) : "memory");
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
            if (c + ahead < n) {
                asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");      // the stage of chunk c-1 has been read: reuse it
                load(c + ahead);
            }
        }
        asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");                    // every store of this CTA is complete
    }
    comm_signal(cd, CH_GRID, E, gridDim.x*gridDim.y);
}

// ---- contiguous ranges to every peer through the TMA engine ----
// One warp-sized CTA per (peer, piece): thread 0 streams `bytes` from src (local) to dst (mapped peer memory) through a
// PUSH_STAGES-deep ring of PUSH_CHUNK-byte stages.  Used for the positions of the owned atoms (after k_integrate) and for
// the partial forces of the atoms a rank does not own (three component planes per peer).
__device__ __forceinline__ void tma_stream(const char* src, char* dst, size_t bytes, unsigned char* ring, unsigned long long* bars) {
    // caller: one thread; src, dst, bytes multiples of 16
    const int n = (int) ((bytes + PUSH_CHUNK - 1)/PUSH_CHUNK);
    if (n == 0) return;
    for (int s = 0; s < PUSH_STAGES; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bars[s])));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    auto chunk_bytes = [&](int c) { const size_t r = bytes - (size_t) c*PUSH_CHUNK; return (unsigned int) (r < (size_t) PUSH_CHUNK ? r : (size_t) PUSH_CHUNK); };
    auto load = [&](int c) {
        const unsigned int bar = smem_u32(&bars[c % PUSH_STAGES]), nb = chunk_bytes(c);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(nb) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"(smem_u32(ring + (size_t) (c % PUSH_STAGES)*PUSH_CHUNK)), "l"(src + (size_t) c*PUSH_CHUNK), "r"(nb), "r"(bar) : "memory");
    };
    const int ahead = PUSH_STAGES - 1;
    for (int c = 0; c < n && c < ahead; c++) load(c);
    for (int c = 0; c < n; c++) {
        mbar_wait(smem_u32(&bars[c % PUSH_STAGES]), (unsigned int) ((c/PUSH_STAGES) & 1));
        asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                     :: "l"(dst + (size_t) c*PUSH_CHUNK), "r"(smem_u32(ring + (size_t) (c % PUSH_STAGES)*PUSH_CHUNK)), "r"(chunk_bytes(c)) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        if (c + ahead < n) {
            asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
            load(c + ahead);
        }
    }
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// positions of the owned atoms -> every peer's posq; then CH_POS (the end of a step's exchange: advances the epoch)
// grid (pieces, world-1)
__global__ void __launch_bounds__(32) k_pos_push(NbDev nb, CommDev cd, IntegDev in, int pieces) {
    extern __shared__ __align__(128) unsigned char ring[];
    __shared__ __align__(8) unsigned long long bars[PUSH_STAGES];
    const unsigned long long E = *cd.epoch + 1ull;
    const int q = (cd.rank + 1 + (int) blockIdx.y) % cd.world;            // staggered: the ranks do not all start with peer 0
    const size_t lo = (size_t) cd.atomLo[cd.rank]*sizeof(float4), hi = (size_t) cd.atomLo[cd.rank + 1]*sizeof(float4);
    const size_t per = (((hi - lo) + pieces - 1)/pieces + PUSH_CHUNK - 1)/PUSH_CHUNK*PUSH_CHUNK;
    const size_t b0 = lo + (size_t) blockIdx.x*per, b1 = b0 + per < hi ? b0 + per : hi;
    if (threadIdx.x == 0 && b0 < b1)
        tma_stream((const char*) nb.posq + b0, cd.peer[q] + cd.offPosq + b0, b1 - b0, ring, bars);
    const bool last = comm_arrive(cd, CH_POS, gridDim.x*gridDim.y);
    if (last && threadIdx.x == 0) {
        // the momentum sums of this rank's atoms (k_integrate left them in cmScratch) go along, then the flag
        if (in.fused && in.cmEveryStep) {
            const unsigned long long step = *in.stepCounter - 1ull;               // k_integrate already advanced the counter
            const double* mine = in.cmScratch + 4*((step + 1ull) % 3ull);
            for (int p = 0; p < cd.world; p++) {
                double* t = (double*) (cd.peer[p] + cd.offCm) + cd.rank*12 + 4*((step + 1ull) % 3ull);
                for (int k = 0; k < 4; k++) t[k] = ((volatile const double*) mine)[k];
            }
        }
        comm_publish(cd, CH_POS, E);
        *cd.posNeed = E;
        *cd.epoch = E;
    }
}

// partial forces of the atoms of every other rank -> that rank's inbox, the three component planes as contiguous ranges;
// the local copies are zeroed by the caller (memset nodes) once this kernel has read them.   grid (3, world-1)
__global__ void __launch_bounds__(32) k_force_push_tma(NbDev nb, CommDev cd) {
    extern __shared__ __align__(128) unsigned char ring[];
    __shared__ __align__(8) unsigned long long bars[PUSH_STAGES];
    const unsigned long long E = *cd.epoch + 1ull;
    const int q = (cd.rank + 1 + (int) blockIdx.y) % cd.world;            // staggered: the ranks do not all start with peer 0
    const int c = blockIdx.x;
    // the range is widened to even atom indices (16-byte granularity of the bulk copy): the extra element is an atom the
    // receiver does not own, whose inbox slot it never reads
    const size_t a0 = (size_t) (cd.atomLo[q] & ~1), a1 = (size_t) ((cd.atomLo[q+1] + 1) & ~1);
    const size_t lo = ((size_t) c*nb.npad + a0)*sizeof(long long), hi = ((size_t) c*nb.npad + a1)*sizeof(long long);
    if (threadIdx.x == 0)
        tma_stream((const char*) nb.force + lo, (char*) win_finbox(cd, q, cd.rank, nb.npad) + lo, hi - lo, ring, bars);
    comm_signal(cd, CH_FORCE, E, gridDim.x*gridDim.y);
}

static int sm_count() {
    static int sms = 0;
    if (!sms) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
    return sms;
}

// B200MD_PUSH_TMA: bit 0 charge-grid slabs, bit 1 partial forces, bit 2 positions through the TMA engine.  Default 1: measured
// at 4 ranks on ApoA1 (profiles/r02_multi_gpu.md) the grid push gains (31 -> 24 us), the force push loses (19.5 -> 24 + 3
// memset nodes) and the position push is even (k_integrate with peer stores 32 us = 11.7 + 20).
static int push_tma_mask() {
    static const int m = getenv("B200MD_PUSH_TMA") ? atoi(getenv("B200MD_PUSH_TMA")) : 1;
    return m;
}
static void ring_attr(const void* f) { cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, PUSH_STAGES*PUSH_CHUNK); }

void launch_force_push(const NbDev& nb, const CommDev& cd, cudaStream_t s) {
    if (cd.world <= 1) return;
    if (push_tma_mask() & 2) {
        static bool attr = false;
        if (!attr) { ring_attr((const void*) k_force_push_tma); attr = true; }
        k_force_push_tma<<<dim3(3, cd.world - 1), 32, PUSH_STAGES*PUSH_CHUNK, s>>>(nb, cd);
        // the pushed partials are consumed: zero the foreign ranges for the next evaluation
        for (int c = 0; c < 3; c++) {
            long long* base = nb.force + (size_t) c*nb.npad;
            if (cd.atomLo[cd.rank] > 0) cudaMemsetAsync(base, 0, sizeof(long long)*(size_t) cd.atomLo[cd.rank], s);
            if (cd.atomLo[cd.rank + 1] < nb.natoms) cudaMemsetAsync(base + cd.atomLo[cd.rank + 1], 0, sizeof(long long)*(size_t) (nb.natoms - cd.atomLo[cd.rank + 1]), s);
        }
        return;
    }
    k_force_push<<<std::min((nb.natoms + 255)/256, 2*sm_count()), 256, 0, s>>>(nb, cd);
}
// positions of the owned atoms to every peer (after k_integrate, which then leaves the position stores and CH_POS to this kernel)
bool pos_push_available() { return (push_tma_mask() & 4) != 0; }
void launch_pos_push(const NbDev& nb, const CommDev& cd, const IntegDev& in, cudaStream_t s) {
    if (cd.world <= 1) return;
    static bool attr = false;
    if (!attr) { ring_attr((const void*) k_pos_push); attr = true; }
    const size_t bytes = (size_t) (cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank])*sizeof(float4);
    const int pieces = (int) std::max<size_t>(1, std::min<size_t>(8, bytes/(4*PUSH_CHUNK)));
    k_pos_push<<<dim3(pieces, cd.world - 1), 32, PUSH_STAGES*PUSH_CHUNK, s>>>(nb, cd, in, pieces);
}
void launch_force_total(const NbDev& nb, const CommDev& cd, cudaStream_t s) {
    if (cd.world <= 1) return;
    const int own = cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank];
    k_force_total<<<std::max(1, std::min((own + 255)/256, 2*sm_count())), 256, 0, s>>>(nb, cd);
    k_final_wait<<<1, 32, 0, s>>>(cd, CH_FINAL);
}
void launch_vel_push(const NbDev& nb, const CommDev& cd, cudaStream_t s) {
    if (cd.world <= 1) return;
    const int own = cd.atomLo[cd.rank + 1] - cd.atomLo[cd.rank];
    k_vel_push<<<std::max(1, std::min((own + 255)/256, 2*sm_count())), 256, 0, s>>>(nb, cd);
    k_final_wait<<<1, 32, 0, s>>>(cd, CH_VEL);
}
void launch_pos_wait(const NbDev& nb, const CommDev& cd, cudaStream_t s) {
    (void) nb;
    if (cd.world <= 1) return;
    k_pos_wait<<<1, 32, 0, s>>>(cd);
}
void launch_grid_push(const PmeDev& pme, const CommDev& cd, cudaStream_t s) {
    if (cd.world <= 1) return;
    const bool useTma = (push_tma_mask() & 1) != 0;
    const size_t planeBytes = (size_t) pme.ny*pme.nz*sizeof(long long);
    if (useTma && planeBytes % 16 == 0) {          // every slab then starts and ends on a 16-byte boundary (window offsets are multiples of 256)
        static bool attr = false;
        if (!attr) { cudaFuncSetAttribute(k_grid_push_tma, cudaFuncAttributeMaxDynamicSharedMemorySize, PUSH_STAGES*PUSH_CHUNK); attr = true; }
        const size_t maxBytes = (size_t) cd.maxPlanes*planeBytes;
        const int chunks = (int) ((maxBytes + PUSH_CHUNK - 1)/PUSH_CHUNK);
        const int per = std::max(4, (chunks + 63)/64);                 // <= 64 CTAs per peer, >= 4 chunks per CTA
        k_grid_push_tma<<<dim3((chunks + per - 1)/per, cd.world - 1), 32, PUSH_STAGES*PUSH_CHUNK, s>>>(pme, cd, per);
        return;
    }
    const size_t slab = (size_t) cd.maxPlanes*pme.ny*pme.nz/2;          // 16-byte elements per peer
    const int bx = (int) std::max<size_t>(1, std::min<size_t>((slab + 255)/256/4, (size_t) (4*sm_count()/(cd.world - 1) + 1)));
    k_grid_push<<<dim3(bx, cd.world - 1), 256, 0, s>>>(pme, cd);
}
