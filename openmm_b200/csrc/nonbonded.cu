// nonbonded.cu -- neighbour-list construction and the direct-space 32x32 tile kernel (sm_90a).
//
// Replaces (reference, platforms/cuda): findBlockBounds/sortBoxData/findBlocksWithInteractions
// (findInteractingBlocks.cu:7,54,180), CudaSort (sort.cu), the host-side Hilbert reorder
// (ComputeContext.cpp:447-612) and computeNonbonded (nonbonded.cu:106-652) with body
// coulombLennardJones.cc:1-116.  Arithmetic follows ReferenceLJCoulombIxn::calculateEwaldIxn
// (ReferenceLJCoulombIxn.cpp:373-460) and calculateOneIxn for the cutoff / no-cutoff methods.
//
// Design (not the reference's): atoms are fully re-sorted on the device along a blocked-serpentine order of binning
// cells every time the list is rebuilt; the tile kernel works on the sorted copy (ListDev::sposq, exact user coordinates)
// while integration/bonded code keeps the user's order.  Exclusion masks are generated on the fly while tiles are
// emitted, so there is no static "exclusion tile" set and no host involvement.  There are two complete lists
// (NbDev::list[2]): a build always fills the one that is not current and flips counters[CT_CUR] on the device.
// A build is two launches, k_list_prep and k_build_tiles, that return at once unless counters[CT_REBUILD] is raised.
// The tile kernel (k_pair) is fp32 with two exceptions that the parity against the Reference platform asked for: pairs closer
// than NbDev::closeCut2 are queued per warp and evaluated in double from the exact coordinates (close_pair_double), and the
// fp32 force sums are folded every 8 terms (the j atoms rotate in four octets): see the comments at pair_tiles.  The tile
// kernel's forces go to a sorted-order buffer (NbDev::forceS) that k_fold_sorted adds into the user-order one.
#include "engine.h"
#include "../../include/b200md.h"
#include <algorithm>

#define FULL 0xffffffffu

// squared distance from the (periodic image of the) point/box centre offset d to an axis-aligned box of half
// extents h centred at the origin.  Orthorhombic: the per-axis nearest image minimises it.  Triclinic: the 3-step
// reduction is not guaranteed to pick the image nearest to the BOX, so all 27 neighbouring images are tried
// (list construction only; the pair kernel applies the reference's own 3-step minimum image per pair).
__device__ __forceinline__ float box_dist2(float3 d, float hx, float hy, float hz, const BoxDev& b, bool periodic) {
    if (periodic) d = min_image(d, b);
    if (!periodic || !b.triclinic) {
        const float dx = fmaxf(0.f, fabsf(d.x) - hx), dy = fmaxf(0.f, fabsf(d.y) - hy), dz = fmaxf(0.f, fabsf(d.z) - hz);
        return dx*dx + dy*dy + dz*dz;
    }
    float best = 3e38f;
    for (int sz = -1; sz <= 1; sz++)
        for (int sy = -1; sy <= 1; sy++)
            for (int sx = -1; sx <= 1; sx++) {
                const float x = d.x + sx*b.ax + sy*b.bx + sz*b.cx;
                const float y = d.y + sy*b.by + sz*b.cy;
                const float z = d.z + sz*b.cz;
                const float dx = fmaxf(0.f, fabsf(x) - hx), dy = fmaxf(0.f, fabsf(y) - hy), dz = fmaxf(0.f, fabsf(z) - hz);
                best = fminf(best, dx*dx + dy*dy + dz*dz);
            }
    return best;
}

// ------------------------------------------------------------------------------------------------
// 1. rebuild decision: any atom moved more than padding/2 since the last build (findInteractingBlocks.cu:67-76), fused
// with the per-step refresh of the sorted position copy (with the CURRENT order; a rebuild in the same step rewrites it).
__global__ void __launch_bounds__(256) k_check_gather(NbDev nb, CommDev cd) {
    comm_wait(cd, CH_POS, cd.world > 1 ? *cd.posNeed : 0ull);      // multi-GPU: the owners' position stores of the last step have landed
    const int s = blockIdx.x*blockDim.x + threadIdx.x;
    const ListDev& L = nb.list[nb.counters[CT_CUR] & 1];
    if (s == 0) { nb.counters[CT_CURSOR] = 0; nb.counters[CT_PAIRSTART] = 0; }       // tile cursor / start count of the SM-partitioned tile kernel
    if (s < nb.natoms) {
        const float4 p = nb.posq[s];
        const float4 r = nb.refPos[s];
        const float dx = p.x-r.x, dy = p.y-r.y, dz = p.z-r.z;
        const float d2 = dx*dx + dy*dy + dz*dz;
        if (!(d2 <= nb.halfPad2))       // also true for NaN
            nb.counters[CT_REBUILD] = 1;
    }
    if (s < nb.npad) {
        int a = L.sorig[s];
        if (a < 0 || a >= nb.natoms) a = L.sorig[nb.natoms-1];
        a = min(max(a, 0), nb.natoms-1);          // garbage-safe before the first build
        float4 p = nb.posq[a];
        if (s >= nb.natoms) p.w = 0.f;
        L.sposq[s] = p;                           // exact user coordinates: the pair kernel picks the image itself
    }
}

// ------------------------------------------------------------------------------------------------
// 1b. molecule wrapping (first phase of a list build).  The user's coordinates are never wrapped by the reference
// (getState without enforcePeriodicBox returns a continuous trajectory), but fp32 coordinates must stay small: a molecule
// whose first atom is more than one box length outside the primary cell is moved back by whole lattice vectors, all its
// atoms together (bonded terms and constraints use no minimum image), and cellOffset records the move.  Molecules within
// one box length are left alone, so a freshly set structure keeps its exact coordinates.
__device__ __forceinline__ void wrap_molecule(const NbDev& nb, int m) {
    const int begin = nb.molStart[m], end = nb.molStart[m+1];
    const float4 p = nb.posq[nb.molAtoms[begin]];
    const double* R = nb.box.recip;
    const double px = p.x - nb.origin[0], py = p.y - nb.origin[1], pz = p.z - nb.origin[2];
    const double f[3] = {px*R[0] + py*R[3] + pz*R[6], px*R[1] + py*R[4] + pz*R[7], px*R[2] + py*R[5] + pz*R[8]};
    int k[3];
    bool move = false;
    for (int d = 0; d < 3; d++) {
        const double w = floor(f[d]);
        k[d] = (w >= 2.0 || w <= -2.0) ? (int) w : 0;          // NaN compares false: no move
        move |= (k[d] != 0);
    }
    if (!move) return;
    const BoxDev& b = nb.box;
    const double sx = -(k[0]*(double) b.dax + k[1]*(double) b.bx + k[2]*(double) b.cx);
    const double sy = -(k[1]*(double) b.dby + k[2]*(double) b.cy);
    const double sz = -(k[2]*(double) b.dcz);
    for (int t = begin; t < end; t++) {
        const int a = nb.molAtoms[t];
        if (nb.posqCorr) {          // mixed precision: hi + lo + shift in double, stored as hi / lo (no rounding to fp32)
            const double4 q = load_pos<double>(nb, a);
            store_pos<double>(nb, a, q.x + sx, q.y + sy, q.z + sz);
        }
        else {
            const float4 q = nb.posq[a];
            nb.posq[a] = make_float4((float) ((double) q.x + sx), (float) ((double) q.y + sy), (float) ((double) q.z + sz), q.w);
        }
        nb.cellOffset[a] += k[0]; nb.cellOffset[a + nb.npad] += k[1]; nb.cellOffset[a + 2*nb.npad] += k[2];
    }
}

// ------------------------------------------------------------------------------------------------
// 2. binning (periodic systems only; non-periodic systems keep the identity order)
__device__ __forceinline__ void bin_atom(const NbDev& nb, int a) {
    float4 p = nb.posq[a];
    int key = 0;
    float4 shift = make_float4(0, 0, 0, 0);
    if (nb.box.periodic) {
        const double* R = nb.box.recip;
        double f[3];
        const double px = p.x - nb.origin[0], py = p.y - nb.origin[1], pz = p.z - nb.origin[2];
        f[0] = px*R[0] + py*R[3] + pz*R[6];
        f[1] = px*R[1] + py*R[4] + pz*R[7];
        f[2] = px*R[2] + py*R[5] + pz*R[8];
        int c[3];
        float fl[3];
        for (int d = 0; d < 3; d++) {
            double w = floor(f[d]);
            fl[d] = (float) w;
            double fr = f[d] - w;
            int ci = (int) (fr*nb.ncell[d]);
            c[d] = min(max(ci, 0), nb.ncell[d]-1);
        }
        shift.x = -(fl[0]*nb.box.ax + fl[1]*nb.box.bx + fl[2]*nb.box.cx);
        shift.y = -(fl[1]*nb.box.by + fl[2]*nb.box.cy);
        shift.z = -(fl[2]*nb.box.cz);
        key = nb.cellRank[(c[0]*nb.ncell[1] + c[1])*nb.ncell[2] + c[2]];
    }
    else
        key = 0;
    nb.atomCell[a] = key;
    nb.atomShift[a] = shift;
    atomicAdd(&nb.cellCount[key], 1);
}

// exclusive prefix sum over the CTA (blockDim.x a multiple of 32, at most 1,024 threads); *total = the CTA's sum.
// ws: 32 ints of shared memory.
__device__ __forceinline__ int block_exclusive_scan(int v, int* ws, int* total) {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    int x = v;
    for (int off = 1; off < 32; off <<= 1) {
        const int y = __shfl_up_sync(FULL, x, off);
        if (lane >= off) x += y;
    }
    if (lane == 31) ws[w] = x;
    __syncthreads();
    if (w == 0) {
        int t = (lane < nw) ? ws[lane] : 0;
        for (int off = 1; off < 32; off <<= 1) {
            const int y = __shfl_up_sync(FULL, t, off);
            if (lane >= off) t += y;
        }
        if (lane < nw) ws[lane] = t;
    }
    __syncthreads();
    const int r = x - v + (w > 0 ? ws[w-1] : 0);
    *total = ws[nw-1];
    __syncthreads();          // ws is reused by the next call
    return r;
}

// exclusive scan of cellCount[0..ncells) into cellCount (in place), by the whole grid: CTA b scans the contiguous slice
// [b*per, (b+1)*per) and adds the sums of the slices before it, which every CTA publishes as soon as it has its own (all
// CTAs are co-resident, so the waits end).  The sums go to tmpSorted[0..G), which the binning phase zeroes (0 = not yet
// published, else sum + 1) and the fill phase overwrites.  ws: 33 ints of shared memory.
__device__ void scan_cells_grid(const NbDev& nb, int* ws) {
    const int n = nb.ncells, per = (n + gridDim.x - 1)/gridDim.x;
    const int begin = min((int) blockIdx.x*per, n), end = min(begin + per, n);
    int* sums = nb.tmpSorted;
    int local = 0;
    for (int i = begin + threadIdx.x; i < end; i += blockDim.x) local += nb.cellCount[i];
    int mine;
    block_exclusive_scan(local, ws, &mine);
    if (threadIdx.x == 0) atomicExch(&sums[blockIdx.x], mine + 1);
    if (threadIdx.x < 32) {
        int before = 0;
        for (int b = threadIdx.x; b < (int) blockIdx.x; b += 32) {
            int v;
            long spins = 0;
            while ((v = *((volatile int*) &sums[b])) == 0) {
                __nanosleep(32);
                if (++spins > (1L << 23)) { nb.counters[CT_OVERFLOW] = 2; v = 1; break; }
            }
            before += v - 1;
        }
        for (int off = 16; off > 0; off >>= 1) before += __shfl_xor_sync(FULL, before, off);
        if (threadIdx.x == 0) ws[32] = before;
    }
    __syncthreads();
    int run = ws[32];
    for (int c0 = begin; c0 < end; c0 += blockDim.x) {
        const int i = c0 + threadIdx.x;
        const int c = (i < end) ? nb.cellCount[i] : 0;
        int chunk;
        const int r = block_exclusive_scan(c, ws, &chunk);
        if (i < end) nb.cellCount[i] = run + r;
        run += chunk;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) nb.cellCount[n] = nb.natoms;
}

__device__ __forceinline__ void fill_atom(const NbDev& nb, int a) {
    int key = nb.atomCell[a];
    int slot = nb.cellCount[key] + atomicAdd(&nb.cellFill[key], 1);
    nb.tmpSorted[slot] = a;
}

__device__ __forceinline__ void finalize_slot(const NbDev& nb, const ListDev& L, int s) {
    if (s < nb.natoms) {
        int a = s;
        if (nb.box.periodic) {
            // fill_atom left the atoms of a cell in arrival order; the order inside a cell is made deterministic here
            // (ascending user index) by ranking the atom among its <= ~10 cell mates instead of sorting the cell
            a = nb.tmpSorted[s];
            const int key = nb.atomCell[a];
            const int begin = nb.cellCount[key], end = nb.cellCount[key+1];
            int rank = 0;
            for (int t = begin; t < end; t++) rank += (nb.tmpSorted[t] < a);
            s = begin + rank;
        }
        float4 p = nb.posq[a];
        float4 sh = nb.atomShift[a];
        L.sorig[s] = a;
        nb.sortedOf[a] = s;
        L.swrap[s] = make_float4(p.x+sh.x, p.y+sh.y, p.z+sh.z, p.w);   // wrapped into the anchored cell: list build only
        L.sposq[s] = p;
        L.ssigeps[s] = nb.sigeps[a];
        L.schargeD[s] = nb.chargeD[a];
        L.ssigepsD[s] = nb.sigepsD[a];
        nb.refPos[a] = p;
        if (s == 0) L.lc[LC_MAXHALF] = 0;        // max block half extent, filled by the block-bounds phase
    }
    else {
        L.sorig[s] = -1;
        L.ssigeps[s] = make_float2(0, 0);
        L.schargeD[s] = 0.0;
        L.ssigepsD[s] = make_double2(0.0, 0.0);
        // position is filled by the block-bounds phase with a copy of a real atom of the same block
    }
}

// ------------------------------------------------------------------------------------------------
// The phases above, then the block and superblock bounding boxes (findBlockBounds, findInteractingBlocks.cu:7-52), run as
// ONE launch, k_list_prep, with software grid barriers between the phases.  Why: a rebuild is needed every
// ~4th step only, and what the other steps pay for it is what a NOT-taken rebuild costs in front of the tile kernel: ~15 us
// of latency for a CUDA-graph IF node, or ~2 us per gated kernel that only reads the flag and returns.  Two gated launches
// (this one and k_build_tiles) cost ~4 us.  The grid is sized to be co-resident (<= 2 CTAs of 256 threads per SM); CTAs
// that find no free slot yet (the charge spreading runs beside it) join late, the others wait for them at the first
// barrier, and every wait is bounded (a time-out raises the sticky error flag instead of hanging the device).
__device__ __forceinline__ void grid_barrier(const NbDev& nb, int target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(&nb.counters[CT_BAR], 1);
        long spins = 0;
        while (*((volatile int*) &nb.counters[CT_BAR]) < target) {
            __nanosleep(32);
            if (++spins > (1L << 23)) { nb.counters[CT_OVERFLOW] = 2; break; }
        }
        __threadfence();
    }
    __syncthreads();
}

__device__ void list_prep_phases(const NbDev& nb, const ListDev& L, int* ws) {
    const int G = gridDim.x;
    const int gtid = blockIdx.x*blockDim.x + threadIdx.x, gthreads = G*blockDim.x;
    const int lane = threadIdx.x & 31, gwarp = gtid >> 5, gwarps = gthreads >> 5;
    // 0. molecules that have walked away come home (rare; the barrier is skipped when wrapping is off)
    int base = 0;
    if (nb.nmol > 0) {
        for (int m = gtid; m < nb.nmol; m += gthreads) wrap_molecule(nb, m);
        grid_barrier(nb, G);
        base = G;
    }
    // 1. binning
    for (int a = gtid; a < nb.natoms; a += gthreads) bin_atom(nb, a);
    if (gtid < G) nb.tmpSorted[gtid] = 0;          // the scan's slice sums (npad >= G)
    grid_barrier(nb, base + G);
    // 2. exclusive scan of the cell counts
    scan_cells_grid(nb, ws);
    grid_barrier(nb, base + 2*G);
    // 3. atoms into their cells
    for (int a = gtid; a < nb.natoms; a += gthreads) fill_atom(nb, a);
    grid_barrier(nb, base + 3*G);
    // 4. deterministic in-cell order, sorted copies
    for (int s = gtid; s < nb.npad; s += gthreads) finalize_slot(nb, L, s);
    grid_barrier(nb, base + 4*G);
    // 5. block bounding boxes (one warp per block); the binning counters are consumed: zero them for the next build
    for (int b = gwarp; b < nb.nblocks; b += gwarps) {
        const int s = b*32 + lane;
        const int sl = min(s, nb.natoms-1);
        const float4 p = L.swrap[sl];
        if (s >= nb.natoms) { L.swrap[s] = make_float4(p.x, p.y, p.z, 0.f); L.sposq[s] = make_float4(p.x, p.y, p.z, 0.f); }
        float lox = p.x, hix = p.x, loy = p.y, hiy = p.y, loz = p.z, hiz = p.z;
        for (int off = 16; off > 0; off >>= 1) {
            lox = fminf(lox, __shfl_xor_sync(FULL, lox, off)); hix = fmaxf(hix, __shfl_xor_sync(FULL, hix, off));
            loy = fminf(loy, __shfl_xor_sync(FULL, loy, off)); hiy = fmaxf(hiy, __shfl_xor_sync(FULL, hiy, off));
            loz = fminf(loz, __shfl_xor_sync(FULL, loz, off)); hiz = fmaxf(hiz, __shfl_xor_sync(FULL, hiz, off));
        }
        if (lane == 0) {
            L.blockCenter[b] = make_float4(0.5f*(lox+hix), 0.5f*(loy+hiy), 0.5f*(loz+hiz), 0);
            L.blockHalf[b] = make_float4(0.5f*(hix-lox), 0.5f*(hiy-loy), 0.5f*(hiz-loz), 0);
            atomicMax(&L.lc[LC_MAXHALF], __float_as_int(0.5f*fmaxf(hix-lox, fmaxf(hiy-loy, hiz-loz))));
        }
    }
    for (int i = gtid; i <= nb.ncells; i += gthreads) {
        nb.cellCount[i] = 0;
        if (i < nb.ncells) nb.cellFill[i] = 0;
    }
    if (gtid < TILE_REGIONS) { L.lc[LC_TILES + gtid] = 0; L.lc[LC_MASKS + gtid] = 0; }
    grid_barrier(nb, base + 5*G);
    // 6. superblock boxes (one warp per 32 blocks)
    const int nsuper = (nb.nblocks + 31) >> 5;
    for (int sb = gwarp; sb < nsuper; sb += gwarps) {
        const int b = sb*32 + lane;
        float lox = 3e38f, hix = -3e38f, loy = 3e38f, hiy = -3e38f, loz = 3e38f, hiz = -3e38f;
        if (b < nb.nblocks) {
            const float4 c = L.blockCenter[b], h = L.blockHalf[b];
            lox = c.x - h.x; hix = c.x + h.x; loy = c.y - h.y; hiy = c.y + h.y; loz = c.z - h.z; hiz = c.z + h.z;
        }
        for (int off = 16; off > 0; off >>= 1) {
            lox = fminf(lox, __shfl_xor_sync(FULL, lox, off)); hix = fmaxf(hix, __shfl_xor_sync(FULL, hix, off));
            loy = fminf(loy, __shfl_xor_sync(FULL, loy, off)); hiy = fmaxf(hiy, __shfl_xor_sync(FULL, hiy, off));
            loz = fminf(loz, __shfl_xor_sync(FULL, loz, off)); hiz = fmaxf(hiz, __shfl_xor_sync(FULL, hiz, off));
        }
        if (lane == 0) {
            L.superCenter[sb] = make_float4(0.5f*(lox+hix), 0.5f*(loy+hiy), 0.5f*(loz+hiz), 0);
            L.superHalf[sb] = make_float4(0.5f*(hix-lox), 0.5f*(hiy-loy), 0.5f*(hiz-loz), 0);
        }
    }
}
// the last CTA to leave re-arms the barrier for the next build
__device__ __forceinline__ void grid_barrier_exit(const NbDev& nb) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(&nb.counters[CT_BAREXIT], 1) == (int) gridDim.x - 1) { nb.counters[CT_BAR] = 0; nb.counters[CT_BAREXIT] = 0; }
    }
}

__global__ void __launch_bounds__(256) k_list_prep(NbDev nb) {
    if (nb.counters[CT_REBUILD] == 0) return;
    const ListDev& L = nb.list[(nb.counters[CT_CUR] & 1) ^ 1];      // the list under construction
    __shared__ int ws[33];
    list_prep_phases(nb, L, ws);
    grid_barrier_exit(nb);
}

#define MAX_CACHED_EXCL 24
#define TILE_SPAN 1024         // sorted-index span of a tile that flush_tile indexes directly (bytes of shared memory per warp)
#define SB_MAX 1024            // superblocks listed per pass of k_build_tiles (1024 superblocks = 1.05 M atoms)
// Emit one tile from the first `count` entries of buf (ascending sorted indices).
// sexc: this lane's exclusion partners as SORTED indices, cached once per i-block (nexc of them; partners beyond
// MAX_CACHED_EXCL are looked up in global memory).  esig: bit (b mod 32) is set for every block b that holds one of them
// (all bits when some are not cached): the partners are only searched in tiles that hold such a block.  slotOf: this warp's
// TILE_SPAN bytes of shared memory, all zero on entry and on return; a tile whose j-slots span fewer than TILE_SPAN
// sorted indices is indexed through it (slotOf[j - first j] = lane + 1), wider ones are searched by bisection.
// Tile slots come from TILE_REGIONS independent sub-pools (i-block ib allocates from pool ib % TILE_REGIONS): one global
// counter would take ~14k (DHFR) to ~66k (ApoA1) returning atomics on ONE address per build, which L2 serialises at ~2 ns
// each.  Pool r owns the slots [r*cap, (r+1)*cap), cap = maxTiles/TILE_REGIONS; consumers flatten the pools with a
// 32-lane prefix sum (tile_cursor below).
__device__ void flush_tile(const NbDev& nb, const ListDev& L, int ib, const int* buf, int count, bool diagonal, int lane,
                           const int* sexc, int nexc, int e0, unsigned int esig, unsigned char* slotOf) {
    const int region = ib % TILE_REGIONS;
    const int cap = nb.maxTiles/TILE_REGIONS;
    int k = 0;
    if (lane == 0) k = atomicAdd(&L.lc[LC_TILES + region], 1);      // the slot is not needed until the mask is formed
    const int myj = (lane < count) ? buf[lane] : -1;
    const unsigned int tsig = __reduce_or_sync(FULL, (lane < count) ? 1u << ((myj >> 5) & 31) : 0u);   // blocks in the tile
    const bool indexed = (buf[count-1] - buf[0] < TILE_SPAN) && (esig & tsig) != 0u;
    if (__any_sync(FULL, indexed)) {
        if (lane < count) slotOf[myj - buf[0]] = (unsigned char) (lane + 1);
        __syncwarp();
    }
    unsigned int valid = (count >= 32) ? FULL : ((1u << count) - 1u);
    unsigned int mask = valid;
    bool need = (count < 32);
    int si = ib*32 + lane;
    if (diagonal) {            // own block against itself: keep j > i only
        unsigned int le = (lane == 31) ? FULL : ((2u << lane) - 1u);
        mask &= ~le;
        need = true;
    }
    if (si >= nb.natoms) { mask = 0; need = true; }
    else if (esig & tsig) {
        const int jlo = buf[0], jhi = buf[count-1];
        if (jhi - jlo < TILE_SPAN) {
            for (int e = 0; e < nexc; e++) {
                const int sj = (e < MAX_CACHED_EXCL) ? sexc[e] : nb.sortedOf[nb.exclList[e0 + e]];
                if (!((tsig >> ((sj >> 5) & 31)) & 1u) || sj < jlo || sj > jhi) continue;
                const int p = slotOf[sj - jlo];
                if (p) { mask &= ~(1u << (p - 1)); need = true; }
            }
        }
        else {
            for (int e = 0; e < nexc; e++) {
                const int sj = (e < MAX_CACHED_EXCL) ? sexc[e] : nb.sortedOf[nb.exclList[e0 + e]];
                if (!((tsig >> ((sj >> 5) & 31)) & 1u) || sj < jlo || sj > jhi) continue;
                int lo = 0, hi = count-1;          // binary search in the ascending tile
                while (lo < hi) { int mid = (lo+hi) >> 1; if (buf[mid] < sj) lo = mid+1; else hi = mid; }
                if (buf[lo] == sj) { mask &= ~(1u << lo); need = true; }
            }
        }
    }
    need = __any_sync(FULL, need);
    if (__any_sync(FULL, indexed)) {
        __syncwarp();
        if (lane < count) slotOf[myj - buf[0]] = 0;
    }
    k = __shfl_sync(FULL, k, 0);
    if (k >= cap) { if (lane == 0) nb.counters[CT_OVERFLOW] = 1; return; }
    const int t = region*cap + k;
    L.tileJ[t*32 + lane] = myj;
    int mi = -1;
    if (need) {             // the mask takes the tile's own slot of maskPool (capacity == maxTiles): no second returning atomic
        if (lane == 0) atomicAdd(&L.lc[LC_MASKS + region], 1);
        mi = t;
        L.maskPool[mi*32 + lane] = mask;
    }
    if (lane == 0) { L.tileI[t] = ib; L.tileMask[t] = mi; }
}

// One CTA (4 warps) per i-block: the candidate j-blocks of the i-block are dealt round-robin to the 4 warps (chunks of
// 32 blocks), each warp culls j-blocks by box distance, then j-atoms against the i-block (box, then exact atom
// distances), compacts survivors into its own 32-wide tiles and flushes full tiles as it goes.  The warps' partial
// buffers are merged, sorted and flushed by warp 0 at the end, so an i-block still ends with at most one partial tile.
// (findBlocksWithInteractions, findInteractingBlocks.cu:180-405, is the reference counterpart.  Round-1 profile: with a
// single warp per i-block the kernel was one long dependent chain of L2 round trips per block, 150 us at DHFR size.)
// end of a list build: the last CTA of k_build_tiles to finish makes the new list current
__device__ __forceinline__ void list_block_done(const NbDev& nb) {
    __threadfence();
    if (atomicAdd(&nb.counters[CT_BTDONE], 1) == (int) gridDim.x - 1) {
        nb.counters[CT_BTDONE] = 0;
        nb.counters[CT_BUILDS] += 1;
        nb.counters[CT_REBUILD] = 0;
        nb.counters[CT_CUR] ^= 1;
    }
}

// shared-memory working set of one i-block under construction (one group of NW warps)
template <int NW>
struct BuildSmem {
    int sbuf[NW][64];
    int sstage[NW][64];                           // j-atoms that passed the box test and wait for the exact cull
    int sexcAll[32][MAX_CACHED_EXCL + 1];         // +1: odd stride, conflict-free per-lane rows
    unsigned int sexcSigPart[NW][32];             // blocks (mod 32) of the partners each warp translated ...
    unsigned int sexcSig[32];                     // ... and of all of a lane's partners (flush_tile's esig)
    float4 sipos[32];                             // the i-block's atoms, relative to the block centre
    int sleft[NW];
    __align__(16) unsigned char sslotOf[NW][TILE_SPAN];          // flush_tile's j-slot -> lane index, kept all zero between flushes
    int sbList[SB_MAX];                           // superblocks within range of this i-block
    int sbCount;
    int smerged[NW*32];
};
// barrier over the NW warps that build one i-block (a named barrier, so that several groups could share a CTA)
__device__ __forceinline__ void group_sync(int barId, int nthreads) {
    asm volatile("bar.sync %0, %1;" :: "r"(barId), "r"(nthreads) : "memory");
}

// All tiles of i-block ib, by a group of NW warps (w = warp within the group).
template <int NW>
__device__ void build_tiles_iblock(const NbDev& nb, const ListDev& L, int ib, int w, int lane, BuildSmem<NW>& S, int barId) {
    int* buf = S.sbuf[w];
    // this lane's exclusion partners, translated to sorted indices ONCE per i-block; the warps share the dependent
    // exclList -> sortedOf look-ups (up to MAX_CACHED_EXCL per lane for protein atoms), warp w taking partners w, w+NW, ..
    int* sexc = S.sexcAll[lane];
    int nexc = 0, e0 = 0;
    {
        const int si = ib*32 + lane;
        unsigned int sig = 0;
        if (si < nb.natoms) {
            const int a = L.sorig[si];
            e0 = nb.exclStart[a];
            nexc = nb.exclStart[a+1] - e0;
            for (int e = w; e < nexc && e < MAX_CACHED_EXCL; e += NW) {
                const int sj = nb.sortedOf[nb.exclList[e0 + e]];
                sexc[e] = sj;
                sig |= 1u << ((sj >> 5) & 31);
            }
            if (nexc > MAX_CACHED_EXCL) sig = FULL;
        }
        S.sexcSigPart[w][lane] = sig;
        for (int i = threadIdx.x; i < NW*TILE_SPAN/16; i += NW*32) reinterpret_cast<int4*>(&S.sslotOf[0][0])[i] = make_int4(0, 0, 0, 0);
    }
    auto flush = [&](const int* tile, int count, bool diagonal) {
        flush_tile(nb, L, ib, tile, count, diagonal, lane, sexc, nexc, e0, S.sexcSig[lane], S.sslotOf[w]);
    };
    const float4 ci = L.blockCenter[ib];
    const float4 hi = L.blockHalf[ib];
    if (w == 0) {
        const float4 p = L.swrap[ib*32 + lane];            // padding slots hold a copy of a real atom of the block
        const float qx = p.x-ci.x, qy = p.y-ci.y, qz = p.z-ci.z;
        S.sipos[lane] = make_float4(qx, qy, qz, qx*qx + qy*qy + qz*qz);
    }
    group_sync(barId, NW*32);
    if (w == 0) {                 // read after the group barrier that opens the superblock pass
        unsigned int sig = 0;
        for (int q = 0; q < NW; q++) sig |= S.sexcSigPart[q][lane];
        S.sexcSig[lane] = sig;
    }
    const bool periodic = nb.box.periodic != 0;
    const bool allPairs = (nb.method == B200MD_NB_NOCUTOFF);
    // same condition as the pair kernel's SHIFT mode (lc[LC_MAXHALF] = max block half extent of THIS build)
    const float minL = fminf(nb.box.ax, fminf(nb.box.by, nb.box.cz));
    const bool exactCull = periodic && !nb.box.triclinic &&
                           (0.5f*minL - nb.cutoff - 2.0f*sqrtf(nb.halfPad2) >= __int_as_float(L.lc[LC_MAXHALF]));
    int nbuf = 0;
    // Exact cull: keep j only if it is within the padded cutoff of at least one atom of the i-block.  Valid because every
    // block satisfies halfExtent <= L/2 - cutoff - padding (exactCull is false otherwise).  |d - q|^2 = |q|^2 - 2 d.q + |d|^2
    // with |q|^2 precomputed: 3 FMA per i-atom.  The 1e-5 margin covers the cancellation error (coordinates are relative to
    // the block centre, |d|, |q| < ~3 nm); keeping a j-atom that is a hair outside the padded cutoff is harmless.
    // The cull runs on FULL warps: atoms that pass the box test are staged (ascending, like buf) and tested 32 at a time
    // (tested per candidate block, only ~13 of 32 lanes would be active in the 32-iteration loop).
    int* stg = S.sstage[w];
    int nstg = 0;
    auto exact_stage = [&](int count) {
        const int sj2 = (lane < count) ? stg[lane] : -1;
        bool inc = false;
        if (sj2 >= 0) {
            const float4 pj = L.swrap[sj2];
            const float3 d = min_image(make_float3(pj.x-ci.x, pj.y-ci.y, pj.z-ci.z), nb.box);
            const float mx = -2.0f*d.x, my = -2.0f*d.y, mz = -2.0f*d.z;
            const float thr = nb.paddedCutoff2*1.00001f - (d.x*d.x + d.y*d.y + d.z*d.z);
            // four i-atoms per step: their loads and FMA chains overlap, and only the step's verdict branches
            for (int k = 0; k < 32; k += 4) {
                bool hit = false;
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const float4 q = S.sipos[k + u];
                    hit |= (fmaf(mx, q.x, fmaf(my, q.y, fmaf(mz, q.z, q.w))) < thr);
                }
                if (hit) { inc = true; break; }
            }
        }
        const unsigned int m = __ballot_sync(FULL, inc);
        const int pos = nbuf + __popc(m & ((1u << lane) - 1u));
        if (inc) buf[pos] = sj2;
        nbuf += __popc(m);
        __syncwarp();
        if (nbuf >= 32) {
            flush(buf, 32, false);
            const int v = (lane + 32 < nbuf) ? buf[lane+32] : 0;
            __syncwarp();
            buf[lane] = v;
            nbuf -= 32;
            __syncwarp();
        }
    };
    // candidate j-blocks are dealt to the 4 warps block by block (jb - ib = 4*(32*it + lane) + w): the neighbours of an
    // i-block cluster in index space, so chunk-wise dealing left three warps waiting at the barrier (48 % of all stall
    // samples in the round-1 profile)
    // Two-level search: warp 0 lists (in ascending order) the superblocks of 32 blocks whose box is within range of the
    // i-block; the blocks of the listed superblocks form the virtual candidate sequence v that is dealt to the warps.
    // (The flat scan over all blocks >= ib was O(blocks^2): 2.9 ms per build at 985k atoms.)
    const int nsuper = (nb.nblocks + 31) >> 5;
    for (int chunk = ib >> 5; chunk < nsuper; chunk += SB_MAX) {
    const int chunkEnd = min(chunk + SB_MAX, nsuper);
    group_sync(barId, NW*32);
    if (w == 0) {
        int cnt = 0;
        for (int s0 = chunk; s0 < chunkEnd; s0 += 32) {
            const int sb = s0 + lane;
            bool ok = false;
            if (sb < chunkEnd) {
                if (allPairs || sb == (ib >> 5)) ok = true;
                else {
                    const float4 cs = L.superCenter[sb];
                    const float4 hs = L.superHalf[sb];
                    const float3 d = make_float3(cs.x-ci.x, cs.y-ci.y, cs.z-ci.z);
                    ok = (box_dist2(d, hi.x+hs.x, hi.y+hs.y, hi.z+hs.z, nb.box, periodic) < nb.paddedCutoff2);
                }
            }
            const unsigned int m = __ballot_sync(FULL, ok);
            if (ok) S.sbList[cnt + __popc(m & ((1u << lane) - 1u))] = sb;
            cnt += __popc(m);
        }
        if (lane == 0) S.sbCount = cnt;
    }
    group_sync(barId, NW*32);
    const int nvirt = S.sbCount*32;
    for (int it = 0; w + NW*32*it < nvirt; it++) {
        const int v = w + NW*(32*it + lane);
        const int jb = (v < nvirt) ? S.sbList[v >> 5]*32 + (v & 31) : nb.nblocks;
        bool cand = false;
        if (jb < nb.nblocks && jb >= ib) {
            if (allPairs || jb == ib) cand = true;
            else {
                float4 cj = L.blockCenter[jb];
                float4 hj = L.blockHalf[jb];
                float3 d = make_float3(cj.x-ci.x, cj.y-ci.y, cj.z-ci.z);
                cand = (box_dist2(d, hi.x+hj.x, hi.y+hj.y, hi.z+hj.z, nb.box, periodic) < nb.paddedCutoff2);
            }
        }
        unsigned int bits = __ballot_sync(FULL, cand);
        while (bits) {
            int b = __ffs(bits) - 1;
            bits &= bits - 1;
            const int vb = w + NW*(32*it + b);
            int jblk = S.sbList[vb >> 5]*32 + (vb & 31);
            int sj = jblk*32 + lane;
            if (exactCull && jblk != ib) {
                bool inb = false;
                if (sj < nb.natoms) {
                    const float4 pj = L.swrap[sj];
                    const float3 d = make_float3(pj.x-ci.x, pj.y-ci.y, pj.z-ci.z);
                    inb = (box_dist2(d, hi.x, hi.y, hi.z, nb.box, periodic) < nb.paddedCutoff2);
                }
                const unsigned int mb = __ballot_sync(FULL, inb);
                const int ps = nstg + __popc(mb & ((1u << lane) - 1u));
                if (inb) stg[ps] = sj;
                nstg += __popc(mb);
                __syncwarp();
                if (nstg >= 32) {
                    exact_stage(32);
                    const int v = (lane + 32 < nstg) ? stg[lane+32] : 0;
                    __syncwarp();
                    stg[lane] = v;
                    nstg -= 32;
                    __syncwarp();
                }
                continue;
            }
            bool inc = false;
            if (sj < nb.natoms) {
                if (allPairs || jblk == ib) inc = true;
                else {
                    float4 pj = L.swrap[sj];
                    float3 d = make_float3(pj.x-ci.x, pj.y-ci.y, pj.z-ci.z);
                    inc = (box_dist2(d, hi.x, hi.y, hi.z, nb.box, periodic) < nb.paddedCutoff2);
                }
            }
            unsigned int m = __ballot_sync(FULL, inc);
            int pos = nbuf + __popc(m & ((1u << lane) - 1u));
            if (inc) buf[pos] = sj;
            nbuf += __popc(m);
            __syncwarp();
            if (jblk == ib) {
                // the diagonal tile is always emitted on its own so that its mask is the simple j>i triangle
                flush(buf, nbuf, true);
                nbuf = 0;
                __syncwarp();
            }
            else if (nbuf >= 32) {
                flush(buf, 32, false);
                int v = (lane + 32 < nbuf) ? buf[lane+32] : 0;
                __syncwarp();
                buf[lane] = v;
                nbuf -= 32;
                __syncwarp();
            }
        }
    }
    }   // superblock chunks
    if (exactCull && nstg > 0) exact_stage(nstg);
    // merge the NW partial buffers (each ascending, < 32 entries): rank sort into S.smerged, flushed by the warps in turn.
    // A value's rank in buffer q is found by binary search (5 steps, not a scan of the whole buffer).
    if (lane == 0) S.sleft[w] = nbuf;
    group_sync(barId, NW*32);
    int total = 0;
    for (int q = 0; q < NW; q++) total += S.sleft[q];
    if (lane < nbuf) {
        const int v = buf[lane];
        int rank = 0;
        for (int q = 0; q < NW; q++) {
            const int* bq = S.sbuf[q];
            int lo = 0, hi = S.sleft[q];
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (bq[mid] < v) lo = mid + 1; else hi = mid; }
            rank += lo;
        }
        S.smerged[rank] = v;                 // sorted indices are unique, so ranks are a permutation
    }
    group_sync(barId, NW*32);
    for (int off = 32*w; off < total; off += 32*NW)
        flush(S.smerged + off, min(32, total - off), false);
    group_sync(barId, NW*32);          // the group's shared memory is reused by its next i-block
}

// at most 48 registers (40 warps per SM): left to itself, ptxas takes 40 and spills in the 4-warp instantiation
template <int NW>
__global__ void __launch_bounds__(NW*32, 40/NW) k_build_tiles(NbDev nb) {
    if (nb.counters[CT_REBUILD] == 0) return;
    if (nb.world > 1 && ((int) blockIdx.x % nb.world) != nb.rank) {           // multi-GPU: tiles of this rank's i-blocks only
        if (threadIdx.x == 0) list_block_done(nb);
        return;
    }
    const ListDev& L = nb.list[(nb.counters[CT_CUR] & 1) ^ 1];      // the list under construction
    __shared__ BuildSmem<NW> S;
    build_tiles_iblock<NW>(nb, L, blockIdx.x, threadIdx.x >> 5, threadIdx.x & 31, S, 1);
    if (threadIdx.x == 0) list_block_done(nb);
}

void launch_check_displacement(const NbDev& nb, const CommDev& cd, cudaStream_t s) {
    k_check_gather<<<(nb.npad+255)/256, 256, 0, s>>>(nb, cd);
}

void launch_list_prep(const NbDev& nb, cudaStream_t s) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    k_list_prep<<<std::max(1, std::min((nb.npad + 255)/256, 2*sms)), 256, 0, s>>>(nb);
}

void launch_build_tiles(const NbDev& nb, cudaStream_t s) {
    // 8 warps per i-block shorten the dependent chain while the grid is under one wave (measured: DHFR 108 -> 98 us per
    // build); above that the extra CTAs only add waves (ApoA1 225 -> 244 us), so large systems keep 4
    if (nb.nblocks <= 1200) k_build_tiles<8><<<nb.nblocks, 256, 0, s>>>(nb);
    else k_build_tiles<4><<<nb.nblocks, 128, 0, s>>>(nb);
}

void launch_list_build(const NbDev& nb, cudaStream_t s) {
    // LIST_BUILD_LAUNCHES kernels, each returns immediately unless counters[CT_REBUILD] is set
    launch_list_prep(nb, s);
    launch_build_tiles(nb, s);
}

// ------------------------------------------------------------------------------------------------
// The direct-space kernel.  One warp per 32x32 tile; lane = i-atom; the 32 j-atoms rotate through the
// lanes by shuffle so every lane sees every j once.  Forces leave the tile as 2^32 fixed point.
//
// Per pair (ReferenceLJCoulombIxn.cpp:388-447), with q pre-multiplied by sqrt(ONE_4PI_EPS0):
//   PME:    dEdR = qi qj/r^3 (erfc(ar) + 2 ar exp(-a^2 r^2)/sqrt(pi)) + sw*eps(12 s^12 - 6 s^6)/r^2 [- E_lj sw'/r]
//           E    = qi qj erfc(ar)/r + sw*eps (s^12 - s^6)
//   cutoff: reaction field (ReferenceLJCoulombIxn.cpp:559-575): dEdR = qi qj (1/r^3 - 2 krf) ..., E = qi qj (1/r + krf r^2 - crf)
//
// The v1 loop was bound by the XU pipe (MUFU + FRND: rsqrt, ex2, rcp and three rintf of the per-pair minimum image =
// 6 XU ops per pair slot).  v2:
//  * SHIFT mode: when every block satisfies halfExtent <= L/2 - cutoff - padding (checked on the device at list
//    build) the j atoms of a tile are moved ONCE to the periodic image nearest the i-block centre, and the per-pair
//    minimum image (3 FRND) disappears; pairs whose true image would differ are beyond the cutoff either way.
//  * the loop body is branch-free (select instead of a divergent branch) so unrolled iterations interleave.
// The fp32 loop evaluates erfc (A&S 7.1.26) with an accurate exp for forces and energy alike.  The identity
// erfc(z) + 2z exp(-z^2)/sqrt(pi) = 1 - z^3 g(z^2), with a (5,5) rational minimax fit of g(w) = (erf(z) - 2z exp(-z^2)/sqrt(pi))/z^3
// on w = z^2 in [0,PME_G_WMAX] (ewald_g, |err| < 1.2e-7 evaluated in fp32), would save a MUFU per pair, but its constant
// ABSOLUTE error of ~1e-7 alpha^3 qq per pair is coherent over neighbour shells (it cost 1e-4 relative on the 894-ion
// fixture), while the exp-based erfc has a RELATIVE error.  Only the double-precision close-pair path uses ewald_g, for the
// small screening term of its force.
#define PME_G_WMAX 14.0f

__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float rsqrt_approx(float x) { float r; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// g(w) = (erf(z) - 2 z exp(-z^2)/sqrt(pi))/z^3, w = z^2 in [0,14]: (5,5) rational fit, |err| < 1.2e-7 in fp32
__device__ __forceinline__ float ewald_g(float w) {
    const float p = fmaf(w, fmaf(w, fmaf(w, fmaf(w, fmaf(w, -3.521083106e-07f, 3.445905357e-05f), 0.0002032837893f), 0.01676110697f), -0.01832553619f), 0.7522528288f);
    const float q = fmaf(w, fmaf(w, fmaf(w, fmaf(w, fmaf(w, 0.0001580620439f, 0.002480551583f), 0.02451798422f), 0.1533710339f), 0.5756407144f), 1.0f);
    return p*rcp_approx(q);
}

// The inner loop was counted in SASS (profiles/r01): v2 spent 96 instructions per pair slot (131 FMUL + 101 FFMA per 4
// slots, denormal/range fix-ups around rsqrtf and __fdividef, switch-function code in the main path).  This version is
// written FMA-first with ftz approximate rcp/rsqrt (one Newton step restores rsqrt to <1 ulp) and moves the switching
// function into its own instantiation: ~58 instructions per slot.
__device__ __forceinline__ float wrap_rel(float p, float c, double L, double invL) {
    double r = (double) p - (double) c;
    r -= L*rint(r*invL);
    return (float) r;
}

// ---- close pairs in double precision ----
// fp32 pair arithmetic has a relative error of ~1.5e-7 and the coordinates relative to the block centre are rounded to
// ~3e-8 nm.  On a hydrogen-bonded pair (|F| ~ 1,500 kJ/mol/nm, dF/dr ~ 16,000) that is 2-5e-4 kJ/mol/nm of absolute error
// on BOTH atoms, which is what an atom with a small net force (a lipid tail atom next to a water, say) is measured
// against in the reference's 1e-4 criterion.  Pairs closer than nb.closeCut (default 0.36 nm, ~6 % of the pairs inside the
// cutoff) are therefore taken out of the fp32 loop: the lane notes (i lane, j slot) in a per-warp queue, and after the 32
// rotations the warp evaluates the queued pairs in double from the EXACT user coordinates and adds the forces to the
// fixed-point buffer directly.  ReferenceLJCoulombIxn.cpp:388-447 (PME) / :559-575 (cutoff) / calculateOneIxn restated.
#define CLOSE_QCAP 96
__device__ __forceinline__ float ewald_g(float w);
template <bool ENERGY, int METHOD, bool SWITCH>
__device__ __forceinline__ void close_pair_double(const NbDev& nb, const ListDev& L, int si, int sj, double& energyD) {
    const float4 a = L.sposq[si], b = L.sposq[sj];
    // parameters in double (sorted copies of the user-order tables): the fp32 copies (q sqrt(k), sigma/2, 2 sqrt(eps)) carry
    // a relative rounding of 6e-8 each, i.e. up to 7e-7 on the r^-12 term of a pair whose force is in the hundreds
    const double qq = L.schargeD[si]*L.schargeD[sj];
    const double2 sa = L.ssigepsD[si], sb = L.ssigepsD[sj];
    double dx = (double) b.x - (double) a.x, dy = (double) b.y - (double) a.y, dz = (double) b.z - (double) a.z;
    const BoxDev& bx = nb.box;
    if (bx.periodic) {
        if (bx.triclinic) {         // ReferenceForce::getDeltaRPeriodic order: c, b, a
            double k = floor(dz*bx.recip[8] + 0.5);
            dx -= k*(double) bx.cx; dy -= k*(double) bx.cy; dz -= k*bx.dcz;
            k = floor(dy*bx.recip[4] + 0.5);
            dx -= k*(double) bx.bx; dy -= k*bx.dby;
            k = floor(dx*bx.recip[0] + 0.5);
            dx -= k*bx.dax;
        }
        else {
            dx -= bx.dax*rint(dx*bx.recip[0]); dy -= bx.dby*rint(dy*bx.recip[4]); dz -= bx.dcz*rint(dz*bx.recip[8]);
        }
    }
    const double r2 = dx*dx + dy*dy + dz*dz;
    const double invR = rsqrt(r2), invR2 = invR*invR;
    double dEdR, e = 0.0;
    if (METHOD == B200MD_NB_PME) {
        // qq/r^3 in double; the Ewald screening term  -qq alpha^3 g(alpha^2 r^2),  g(w) = (erf z - 2 z exp(-z^2)/sqrt(pi))/z^3,
        // is a fifth of it at most for r < 0.32 nm and smooth: the fp32 rational fit of g (|err| 1.2e-7) leaves < 4e-5 kJ/mol/nm
        const float w = nb.alpha*nb.alpha*(float) r2;
        const double a3 = (double) nb.alpha*(double) nb.alpha*(double) nb.alpha;
        if (w < PME_G_WMAX && !ENERGY) dEdR = qq*(invR*invR2 - a3*(double) ewald_g(w));
        else {
            const double ar = (double) nb.alpha*r2*invR;
            const double ec = erfc(ar), ex = exp(-ar*ar);
            dEdR = qq*invR*invR2*(ec + 1.12837916709551257390*ar*ex);
            e = qq*invR*ec;
        }
    }
    else if (METHOD == B200MD_NB_NOCUTOFF) { dEdR = qq*invR*invR2; e = qq*invR; }
    else { dEdR = qq*(invR*invR2 - 2.0*(double) nb.krf); e = qq*(invR + (double) nb.krf*r2 - (double) nb.crf); }
    const double sig = sa.x + sb.x, eps = sa.y*sb.y;
    const double s2 = sig*sig*invR2, s6 = s2*s2*s2;
    double ljF = eps*s6*invR2*(12.0*s6 - 6.0), ljE = eps*s6*(s6 - 1.0);
    if (SWITCH) {
        const double r = r2*invR;
        if (r > (double) nb.switchDist) {
            const double swInv = 1.0/((double) nb.cutoff - (double) nb.switchDist);
            const double x = (r - (double) nb.switchDist)*swInv;
            const double sw = 1.0 + x*x*x*(-10.0 + x*(15.0 - x*6.0));
            const double dsw = x*x*(-30.0 + x*(60.0 - x*30.0))*swInv;
            ljF = sw*ljF - ljE*dsw*invR;
            ljE *= sw;
        }
    }
    dEdR += ljF;
    if (ENERGY) energyD += e + ljE;
    const long long fx = __double2ll_rn(dx*dEdR*B200MD_FORCE_SCALE), fy = __double2ll_rn(dy*dEdR*B200MD_FORCE_SCALE), fz = __double2ll_rn(dz*dEdR*B200MD_FORCE_SCALE);
    atomicAdd((unsigned long long*) &nb.forceS[si], (unsigned long long) (-fx));
    atomicAdd((unsigned long long*) &nb.forceS[si + nb.npad], (unsigned long long) (-fy));
    atomicAdd((unsigned long long*) &nb.forceS[si + 2*nb.npad], (unsigned long long) (-fz));
    atomicAdd((unsigned long long*) &nb.forceS[sj], (unsigned long long) fx);
    atomicAdd((unsigned long long*) &nb.forceS[sj + nb.npad], (unsigned long long) fy);
    atomicAdd((unsigned long long*) &nb.forceS[sj + 2*nb.npad], (unsigned long long) fz);
}

template <bool ENERGY, int METHOD, bool SHIFT, bool SWITCH, bool CLOSE>
__device__ __forceinline__ void pair_tiles(const NbDev& nb, const ListDev& L, float& energy, unsigned short* cq) {
    const int lane = threadIdx.x & 31;
    const int gwarp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x*blockDim.x) >> 5;
    TileCursor cursor;
    cursor.init(nb, L, lane);
    const int ntiles = cursor.total;
    const bool periodic = nb.box.periodic != 0;
    const float cutoff2 = nb.cutoff2;
    const float swInv = SWITCH ? 1.0f/(nb.cutoff - nb.switchDist) : 0.f;
    // Rotation schedule: the 32 j atoms of a tile visit the lanes in four groups of eight.  Inside a group the j atoms rotate
    // through the 8 lanes of their octet; after 8 steps every j is back in its lane, the group's partial forces are folded
    // into running totals, and the octets move on by 8 lanes.  The fp32 accumulators therefore never hold more than 8
    // contributions before they are folded: the rounding of a sum of 32 terms whose partial sums reach hundreds of
    // kJ/mol/nm was the largest remaining error of the fp32 path (profiles/r02_parity_probe.md).
    const int srcIn = (lane & ~7) | ((lane + 1) & 7);
    const int srcOut = (lane + 8) & 31;
    const int sub = lane & 7;
    const float close2 = CLOSE ? nb.closeCut2 : 0.f;
    const unsigned int ltMask = (1u << lane) - 1u;
    double energyD = 0.0;
    // multi-GPU force decomposition: rank r owns the tiles of i-blocks with ib % world == r.  (Tile INDICES are handed out
    // by an atomic counter and differ between ranks; the i-block of a tile does not.)
    __shared__ int sbase;
    int f = gwarp;
    const int wib = threadIdx.x >> 5, wpb = blockDim.x >> 5;
    if (nb.smPartition) f = ntiles;
    for (;; f += nwarps) {
        if (nb.smPartition) {
            // one cursor fetch per CTA and round: CTAs that start late (SM slots held by other kernels) take less work
            __syncthreads();
            if (threadIdx.x == 0) sbase = atomicAdd(&nb.counters[CT_CURSOR], wpb);
            __syncthreads();
            f = sbase + wib;
            if (sbase >= ntiles) break;
            if (f >= ntiles) continue;
        }
        else if (f >= ntiles) break;
        const int t = cursor.slot(f);
        const int ib = L.tileI[t];
        if (nb.world > 1 && (ib % nb.world) != nb.rank) continue;
        const int si = ib*32 + lane;
        float4 pi = L.sposq[si];
        const float2 sei = L.ssigeps[si];
        const int jidx = L.tileJ[t*32 + lane];
        const int jj = max(jidx, 0);
        float4 pj = L.sposq[jj];
        float2 sej = L.ssigeps[jj];
        const int mi = L.tileMask[t];
        const unsigned int mask32 = (mi < 0) ? FULL : L.maskPool[mi*32 + lane];
        if (SHIFT) {
            // single-image mode: coordinates relative to the i-block centre, image chosen ONCE per atom and tile, in
            // double from the exact user coordinates (a lattice shift applied in fp32 costs half an ulp of the box
            // length, ~5e-7 nm: 1e-3 relative on weakly loaded atoms).  The rounding left is that of the ~1 nm relative
            // coordinate (<= 6e-8 nm).
            const float4 c = L.blockCenter[ib];
            const BoxDev& bx = nb.box;
            pi.x = wrap_rel(pi.x, c.x, bx.dax, bx.recip[0]); pi.y = wrap_rel(pi.y, c.y, bx.dby, bx.recip[4]); pi.z = wrap_rel(pi.z, c.z, bx.dcz, bx.recip[8]);
            pj.x = wrap_rel(pj.x, c.x, bx.dax, bx.recip[0]); pj.y = wrap_rel(pj.y, c.y, bx.dby, bx.recip[4]); pj.z = wrap_rel(pj.z, c.z, bx.dcz, bx.recip[8]);
        }
        float fiTx = 0.f, fiTy = 0.f, fiTz = 0.f, fjTx = 0.f, fjTy = 0.f, fjTz = 0.f;
        int qn = 0;
#pragma unroll 1
        for (int g = 0; g < 4; g++) {
        // j slots of this group: octet ((lane >> 3) + g) & 3, starting at this lane's position in the octet
        const int slotBase = (((lane >> 3) + g) & 3) << 3;
        unsigned int mask = (mask32 >> slotBase) & 0xffu;
        mask = ((mask | (mask << 8)) >> sub) & 0xffu;          // bit 0 = the slot held now, bit k = after k rotations
        float fix = 0.f, fiy = 0.f, fiz = 0.f, fjx = 0.f, fjy = 0.f, fjz = 0.f;
#pragma unroll 4
        for (int k = 0; k < 8; k++) {
            float3 d = make_float3(pj.x-pi.x, pj.y-pi.y, pj.z-pi.z);
            if (!SHIFT && periodic) d = min_image(d, nb.box);
            const float r2raw = fmaf(d.z, d.z, fmaf(d.y, d.y, d.x*d.x));
            bool valid = (mask & 1u) && r2raw < cutoff2;
            mask >>= 1;
            if (CLOSE) {
                const bool isClose = valid && r2raw < close2;
                const unsigned int cm = __ballot_sync(FULL, isClose);
                if (cm) {           // warp-uniform; ~1 rotation in 8 at water density
                    const int pos = qn + __popc(cm & ltMask);
                    if (isClose && pos < CLOSE_QCAP) { cq[pos] = (unsigned short) (lane | ((slotBase | ((sub + k) & 7)) << 5)); valid = false; }
                    qn = min(CLOSE_QCAP, qn + __popc(cm));
                }
            }
            const float r2 = valid ? r2raw : 1.0f;
            float y = rsqrt_approx(r2);
            y = y*fmaf(-0.5f*r2, y*y, 1.5f);             // Newton step: F ~ invR^3 needs a <1 ulp invR
            const float invR2 = y*y;
            const float qq = pi.w*pj.w;
            float dEdR, e = 0.f;
            if (METHOD == B200MD_NB_PME) {
                const float r = r2*y;
                const float ar = nb.alpha*r;
                // accurate expf, not __expf: the ex2.approx form loses ulps with |ar^2| and pushed ApoA1 atoms whose net
                // force is a small difference of large direct and reciprocal parts over 1e-4 (no measurable cost here)
                const float ex = expf(-ar*ar);
                // erfc: Abramowitz-Stegun 7.1.26, |err| < 1.5e-7 (same form as coulombLennardJones.cc:15-20)
                const float tt = rcp_approx(fmaf(0.3275911f, ar, 1.0f));
                const float erfcAr = (0.254829592f+(-0.284496736f+(1.421413741f+(-1.453152027f+1.061405429f*tt)*tt)*tt)*tt)*tt*ex;
                const float pref = qq*y;
                dEdR = pref*invR2*fmaf(1.1283791671f*ar, ex, erfcAr);
                e = pref*erfcAr;
            }
            else if (METHOD == B200MD_NB_NOCUTOFF) {
                const float pref = qq*y;
                dEdR = pref*invR2;
                e = pref;
            }
            else {   // cutoff with reaction field
                dEdR = qq*fmaf(-2.0f, nb.krf, y*invR2);
                e = qq*(fmaf(nb.krf, r2, y) - nb.crf);
            }
            const float sig = sei.x + sej.x;
            const float eps = sei.y*sej.y;
            const float s2 = sig*sig*invR2;
            const float s6 = s2*s2*s2;
            const float es6 = eps*s6;
            float ljF = es6*invR2*fmaf(12.0f, s6, -6.0f);
            float ljE = fmaf(es6, s6, -es6);
            if (SWITCH) {
                const float r = r2*y;
                if (r > nb.switchDist) {
                    const float x = (r - nb.switchDist)*swInv;
                    const float sw = 1.0f + x*x*x*(-10.0f + x*(15.0f - x*6.0f));
                    const float dsw = x*x*(-30.0f + x*(60.0f - x*30.0f))*swInv;
                    ljF = sw*ljF - ljE*dsw*y;
                    ljE *= sw;
                }
            }
            dEdR = valid ? dEdR + ljF : 0.f;
            if (ENERGY) energy += valid ? e + ljE : 0.f;
            fix = fmaf(-d.x, dEdR, fix); fiy = fmaf(-d.y, dEdR, fiy); fiz = fmaf(-d.z, dEdR, fiz);
            fjx = fmaf(d.x, dEdR, fjx); fjy = fmaf(d.y, dEdR, fjy); fjz = fmaf(d.z, dEdR, fjz);
            pj.x = __shfl_sync(FULL, pj.x, srcIn); pj.y = __shfl_sync(FULL, pj.y, srcIn);
            pj.z = __shfl_sync(FULL, pj.z, srcIn); pj.w = __shfl_sync(FULL, pj.w, srcIn);
            sej.x = __shfl_sync(FULL, sej.x, srcIn); sej.y = __shfl_sync(FULL, sej.y, srcIn);
            fjx = __shfl_sync(FULL, fjx, srcIn); fjy = __shfl_sync(FULL, fjy, srcIn); fjz = __shfl_sync(FULL, fjz, srcIn);
        }
        // the octet is home again: fold the group's sums, then the j atoms (with their totals) move on by one octet
        fiTx += fix; fiTy += fiy; fiTz += fiz;
        fjTx += fjx; fjTy += fjy; fjTz += fjz;
        pj.x = __shfl_sync(FULL, pj.x, srcOut); pj.y = __shfl_sync(FULL, pj.y, srcOut);
        pj.z = __shfl_sync(FULL, pj.z, srcOut); pj.w = __shfl_sync(FULL, pj.w, srcOut);
        sej.x = __shfl_sync(FULL, sej.x, srcOut); sej.y = __shfl_sync(FULL, sej.y, srcOut);
        fjTx = __shfl_sync(FULL, fjTx, srcOut); fjTy = __shfl_sync(FULL, fjTy, srcOut); fjTz = __shfl_sync(FULL, fjTz, srcOut);
        }   // groups

        if (CLOSE && qn > 0) {
            __syncwarp();
            for (int e = lane; e < qn; e += 32) {
                const int code = cq[e];
                close_pair_double<ENERGY, METHOD, SWITCH>(nb, L, ib*32 + (code & 31), L.tileJ[t*32 + (code >> 5)], energyD);
            }
            __syncwarp();
        }
        // after 4 x 8 rotations every lane holds its own j again.  The totals go to the SORTED-order buffer: the warp's 32
        // i-atoms are one contiguous run per component and the j-atoms of a tile ascend, so the atomics of a warp land on
        // a few L2 lines instead of 32 scattered ones (k_fold_sorted moves them to user order once per evaluation)
        if (si < nb.natoms) {
            atomicAdd((unsigned long long*) &nb.forceS[si], (unsigned long long) float_to_fixed(fiTx));
            atomicAdd((unsigned long long*) &nb.forceS[si + nb.npad], (unsigned long long) float_to_fixed(fiTy));
            atomicAdd((unsigned long long*) &nb.forceS[si + 2*nb.npad], (unsigned long long) float_to_fixed(fiTz));
        }
        if (jidx >= 0) {
            atomicAdd((unsigned long long*) &nb.forceS[jidx], (unsigned long long) float_to_fixed(fjTx));
            atomicAdd((unsigned long long*) &nb.forceS[jidx + nb.npad], (unsigned long long) float_to_fixed(fjTy));
            atomicAdd((unsigned long long*) &nb.forceS[jidx + 2*nb.npad], (unsigned long long) float_to_fixed(fjTz));
        }
    }
    if (ENERGY && CLOSE && energyD != 0.0) atomicAdd(&nb.energy[EN_NB], energyD);
}

template <bool ENERGY, int METHOD, bool SHIFT>
__device__ __forceinline__ void pair_tiles_sw(const NbDev& nb, const ListDev& L, float& energy, unsigned short* cq) {
    if (nb.closeCut2 > 0.f) {
        if (nb.useSwitch) pair_tiles<ENERGY, METHOD, SHIFT, true, true>(nb, L, energy, cq);
        else pair_tiles<ENERGY, METHOD, SHIFT, false, true>(nb, L, energy, cq);
    }
    else {
        if (nb.useSwitch) pair_tiles<ENERGY, METHOD, SHIFT, true, false>(nb, L, energy, cq);
        else pair_tiles<ENERGY, METHOD, SHIFT, false, false>(nb, L, energy, cq);
    }
}

template <bool ENERGY, int METHOD>
__global__ void __launch_bounds__(256, ENERGY ? 2 : 4) k_pair(NbDev nb) {
    if (nb.smPartition) {
        // SM partition (launch_pair_m): CTAs that land on an SM reserved for the reciprocal-space kernels do no tile work.
        // They must not leave at once, though: a reserved SM would then swallow the grid's still-pending CTAs one after the
        // other (each finds room there and exits) while the other SMs are still busy with the charge spreading, and the
        // tile kernel would be left with a fraction of its workers.  So they hold their slots until EVERY CTA of the grid
        // has started (the pending ones can then only have gone to the other SMs), and only then hand the SM over.
        unsigned int smid;
        asm("mov.u32 %0, %%smid;" : "=r"(smid));
        const bool reserved = (nb.pmeSmMask[(smid >> 6) & 3] >> (smid & 63)) & 1ull;
        if (threadIdx.x == 0) {
            atomicAdd(&nb.counters[CT_PAIRSTART], 1);
            if (reserved) {
                long spins = 0;
                while (*((volatile int*) &nb.counters[CT_PAIRSTART]) < (int) gridDim.x && ++spins < (1L << 20)) __nanosleep(200);
            }
        }
        if (reserved) { __syncthreads(); return; }
    }
    float energy = 0.f;
    __shared__ unsigned short closeQ[8][CLOSE_QCAP];       // per-warp queue of close pairs: i lane | j slot << 5
    unsigned short* cq = closeQ[threadIdx.x >> 5];
    const ListDev& L = nb.list[nb.counters[CT_CUR] & 1];
    const float maxHalf = __int_as_float(L.lc[LC_MAXHALF]);       // max block half extent recorded at list build
    const BoxDev& b = nb.box;
    const float minL = fminf(b.ax, fminf(b.by, b.cz));
    const bool shiftOK = b.periodic && !b.triclinic && (0.5f*minL - nb.cutoff - 2.0f*sqrtf(nb.halfPad2) >= maxHalf);
    if (shiftOK) pair_tiles_sw<ENERGY, METHOD, true>(nb, L, energy, cq);
    else pair_tiles_sw<ENERGY, METHOD, false>(nb, L, energy, cq);
    if (ENERGY) {
        for (int off = 16; off > 0; off >>= 1) energy += __shfl_xor_sync(FULL, energy, off);
        if ((threadIdx.x & 31) == 0 && energy != 0.f) atomicAdd(&nb.energy[EN_NB], (double) energy);
    }
}

template <bool ENERGY>
static void launch_pair_m(const NbDev& nb, cudaStream_t s) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    // M waves of short-lived CTAs instead of one wave of persistent ones: SM slots are handed back while the kernel runs.
    // On one GPU the reciprocal-space chain and the bonded terms are graph nodes of a higher priority (launch_high, and the
    // step graph is instantiated with cudaGraphInstantiateFlagUseNodePriority); the FFT, gather and bonded CTAs fit one
    // such slot (in registers; shared memory through pair_set_carveout), so they take the slots as they come free and run
    // inside the tile kernel's span rather than after it.  The spread brick takes two slots.
    const int waves = 4, perSm = 4;
    dim3 grid(sms*perSm*(nb.smPartition ? 1 : waves)), block(256);       // partitioned: ONE persistent wave, tiles from the cursor
    switch (nb.method) {
        case B200MD_NB_PME: k_pair<ENERGY, B200MD_NB_PME><<<grid, block, 0, s>>>(nb); break;
        case B200MD_NB_NOCUTOFF: k_pair<ENERGY, B200MD_NB_NOCUTOFF><<<grid, block, 0, s>>>(nb); break;
        default: k_pair<ENERGY, B200MD_NB_CUTOFF_PERIODIC><<<grid, block, 0, s>>>(nb); break;
    }
}

// Shared-memory carve-out of the PME tile kernel.  Left to itself the driver may configure an SM that runs four tile CTAs
// (a few KiB of shared memory each) with a small carve-out; a chain CTA that needs tens of KiB could then join that SM only
// after it drained and was reconfigured, and while such a high-priority CTA waits, SMs drain for it.  An FFT CTA (fftSmem
// bytes, at most 16,384 registers) joins an SM as soon as one tile CTA retires, so it needs room beside three tile CTAs;
// a spread-brick CTA (brickSmem bytes, 20,480 registers) joins once two have retired, beside two.  Ask for the larger of
// the two; a percentage between two supported capacities selects the larger one.
void pair_set_carveout(size_t fftSmem, size_t brickSmem) {
    int dev = 0, perSm = 0, reserved = 0;
    CUDA_CHECK(cudaGetDevice(&dev));
    CUDA_CHECK(cudaDeviceGetAttribute(&perSm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev));
    CUDA_CHECK(cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev));
    const void* kernels[] = {(const void*) k_pair<false, B200MD_NB_PME>, (const void*) k_pair<true, B200MD_NB_PME>};
    for (const void* k : kernels) {
        cudaFuncAttributes fa;
        CUDA_CHECK(cudaFuncGetAttributes(&fa, k));
        const size_t tile = fa.sharedSizeBytes + reserved;
        const size_t need = std::max(3*tile + fftSmem, 2*tile + brickSmem) + reserved;
        const int percent = std::min(100, (int) ((100*need + perSm - 1)/perSm));
        CUDA_CHECK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, percent));
    }
}

// which SM ids exist (they need not be contiguous): one CTA per resident slot writes its %smid into a bitmap
__global__ void k_smid_probe(unsigned long long* bitmap) {
    unsigned int smid;
    asm("mov.u32 %0, %%smid;" : "=r"(smid));
    if (threadIdx.x == 0) atomicOr(&bitmap[(smid >> 6) & 3], 1ull << (smid & 63));
    // stay resident a little so that the grid spreads over every SM
    const long long t0 = clock64();
    while (clock64() - t0 < 20000) { }
}
// choose `reserve` SMs (the highest ids) for the reciprocal-space chain; returns the number actually reserved
int choose_pme_sms(int reserve, unsigned long long mask[4]) {
    mask[0] = mask[1] = mask[2] = mask[3] = 0ull;
    if (reserve <= 0) return 0;
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    unsigned long long* d = nullptr;
    unsigned long long h[4] = {0, 0, 0, 0};
    if (cudaMalloc(&d, sizeof(h)) != cudaSuccess) return 0;
    cudaMemset(d, 0, sizeof(h));
    k_smid_probe<<<sms*16, 128>>>(d);
    cudaMemcpy(h, d, sizeof(h), cudaMemcpyDeviceToHost);
    cudaFree(d);
    int found = 0, taken = 0;
    for (int w = 0; w < 4; w++) found += __builtin_popcountll(h[w]);
    if (found < sms) return 0;                        // the probe did not see every SM: do not partition
    reserve = std::min(reserve, found/2);
    for (int id = 255; id >= 0 && taken < reserve; id--)
        if ((h[id >> 6] >> (id & 63)) & 1ull) { mask[id >> 6] |= 1ull << (id & 63); taken++; }
    return taken;
}

// The tile kernel's forces, sorted order -> user order: one thread per sorted slot of the list k_pair read.  Atomic, because
// the gather and the bonded terms may be adding to `force` on other streams; forceS is left zeroed for the next evaluation.
__global__ void __launch_bounds__(256) k_fold_sorted(NbDev nb) {
    const int s = blockIdx.x*blockDim.x + threadIdx.x;
    if (s >= nb.natoms) return;
    const ListDev& L = nb.list[nb.counters[CT_CUR] & 1];
    const int a = L.sorig[s];
    for (int c = 0; c < 3; c++) {
        const long long v = nb.forceS[s + c*nb.npad];
        if (v != 0) {
            atomicAdd((unsigned long long*) &nb.force[a + c*nb.npad], (unsigned long long) v);
            nb.forceS[s + c*nb.npad] = 0;
        }
    }
}

void launch_pair(const NbDev& nb, bool energy, cudaStream_t s) {
    if (energy) launch_pair_m<true>(nb, s); else launch_pair_m<false>(nb, s);
    k_fold_sorted<<<(nb.natoms + 255)/256, 256, 0, s>>>(nb);
}

// diagnostic: number of pairs inside the true cutoff that the list evaluates (tile efficiency accounting)
__global__ void k_count_pairs(NbDev nb) {
    const ListDev& L = nb.list[nb.counters[CT_CUR] & 1];
    const int lane = threadIdx.x & 31;
    const int gwarp = (blockIdx.x*blockDim.x + threadIdx.x) >> 5;
    const int nwarps = (gridDim.x*blockDim.x) >> 5;
    TileCursor cursor;
    cursor.init(nb, L, lane);
    const int ntiles = cursor.total;
    if (gwarp == 0 && lane == 0) L.lc[LC_USED] = ntiles;
    int count = 0;
    for (int f = gwarp; f < ntiles; f += nwarps) {
        const int t = cursor.slot(f);
        const int si = L.tileI[t]*32 + lane;
        const float4 pi = L.sposq[si];
        const int mi = L.tileMask[t];
        const unsigned int mask = (mi < 0) ? FULL : L.maskPool[mi*32 + lane];
        for (int k = 0; k < 32; k++) {
            int jidx = L.tileJ[t*32 + k];
            if (jidx < 0 || !((mask >> k) & 1u)) continue;
            float4 pj = L.sposq[jidx];
            float3 d = make_float3(pj.x-pi.x, pj.y-pi.y, pj.z-pi.z);
            if (nb.box.periodic) d = min_image(d, nb.box);
            if (d.x*d.x + d.y*d.y + d.z*d.z < nb.cutoff2) count++;
        }
    }
    for (int off = 16; off > 0; off >>= 1) count += __shfl_xor_sync(FULL, count, off);
    if (lane == 0 && count) atomicAdd(&nb.counters[CT_PAIRS], count);
}

void launch_count_pairs(const NbDev& nb, cudaStream_t s) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaMemsetAsync(&nb.counters[CT_PAIRS], 0, sizeof(int), s);
    k_count_pairs<<<sms*4, 256, 0, s>>>(nb);
}
