// engine.h -- internal declarations shared by the CUDA translation units of libb200md.so.
// Public boundary: include/b200md.h.  Data layout and kernel inventory: DESIGN.md.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdexcept>
#include <string>
#include <vector>

#define B200MD_TILE 32
#define B200MD_PME_ORDER 5           // ReferenceLJCoulombIxn.cpp:243 (pme_init(..., 5, 1)); same on every reference platform
#define B200MD_FORCE_SCALE 4294967296.0   // 2^32 fixed point, as the reference GPU platforms (nonbonded.cu:301-316)
#define B200MD_ONE_4PI_EPS0 138.93545764438198    // SimTKOpenMMRealType.h:89
#define B200MD_BOLTZ 0.00831446261815324  // kJ/mol/K, SimTKOpenMMRealType.h:76-80 (CODATA 2018)
#define B200MD_MAX_RADIX 16
#define B200MD_MAX_FFT_STAGES 8

#define CUDA_CHECK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) throw std::runtime_error(std::string(#x) + ": " + cudaGetErrorString(e_)); } while (0)

// Launch at the device's greatest stream priority, carried by the launch (cudaLaunchAttributePriority) rather than by the
// stream, so that a node captured into a step graph keeps it: the single-GPU step graph is instantiated with
// cudaGraphInstantiateFlagUseNodePriority.  The reciprocal-space chain and the bonded terms launch this way; the CTA
// dispatcher then gives them the SM slots that retiring tile-kernel CTAs hand back before the tile kernel's queued CTAs.
// Elsewhere the attribute changes nothing that matters: multi-GPU graphs are instantiated without the flag, so their nodes
// run at the launch stream's priority as before, and outside graphs these kernels either run on the high-priority
// reciprocal-space stream already or sit in one stream behind the kernels they depend on.
template <typename... P, typename... A>
inline void launch_high(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, A... args) {
    static const int hi = [] { int lo = 0, h = 0; cudaDeviceGetStreamPriorityRange(&lo, &h); return h; }();
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributePriority;
    at[0].val.priority = hi;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
    cfg.attrs = at; cfg.numAttrs = 1;
    CUDA_CHECK(cudaLaunchKernelEx(&cfg, kernel, args...));
}

// Periodic box, reduced lower-triangular form (ContextImpl.cpp:267-275): a=(ax,0,0) b=(bx,by,0) c=(cx,cy,cz).
struct BoxDev {
    float ax, bx, by, cx, cy, cz;
    float invAx, invBy, invCz;
    int triclinic;
    int periodic;
    double dax, dby, dcz;   // box lengths in double (orthorhombic single-image wrap of the pair kernel)
    double recip[9];     // recipBoxVectors[i][j] at recip[3*i+j], as invert_box_vectors (ReferencePME.cpp:196-204)
    double volume;
};

// precision of the spectral pipeline (charge grid -> FFT -> convolution -> potential grid); the input grid is int64
// fixed point either way.  fp32 is sufficient: a double pipeline (make dbl) changes the reciprocal-space force error by
// nothing on DHFR, ApoA1 and the 894-ion fixture.  What DID matter is the precision of the B-spline weights in spreading
// and interpolation, which are double (pme.cu; profiles/r02_parity_probe.md).
#ifdef B200MD_REAL_DOUBLE      // experiment build (make dbl -> libb200md_dbl.so): double spectral pipeline, for error attribution only
typedef double real;
typedef double2 real2;
#else
typedef float real;
typedef float2 real2;
#endif

struct FftPlanDev {      // 1-D mixed-radix Stockham plan for one grid dimension
    int n;
    int nstages;
    int radix[B200MD_MAX_FFT_STAGES];
    const real2* tw;     // tw[k] = exp(-2 pi i k / n), k < n
};

// Everything the force kernels need, passed by value.
// One neighbour list: the sorted copy of the atoms, the 32-atom blocks and the 32x32 tiles.
struct ListDev {
    float4* sposq;               // sorted positions (exact user coordinates, refreshed every step) + charge
    float2* ssigeps;
    double* schargeD;            // sorted copies of NbDev::chargeD / sigepsD (the double-precision close-pair path)
    double2* ssigepsD;
    float4* swrap;               // sorted positions wrapped into the anchored cell at the build (list build only)
    int* sorig;                  // sorted slot -> user atom (-1 for padding)
    float4* blockCenter;
    float4* blockHalf;
    float4* superCenter;         // bounding boxes of superblocks of 32 consecutive blocks (first level of the candidate search)
    float4* superHalf;
    int* tileI;                  // [maxTiles]
    int* tileJ;                  // [maxTiles*32]
    int* tileMask;               // [maxTiles] index into maskPool or -1
    unsigned int* maskPool;      // [maxTiles*32]
    int* lc;                     // per-list counters, LC_* below
};
#define TILE_REGIONS 32
// ListDev::lc: tile and mask-tile counts of the TILE_REGIONS slot pools, max block half extent (float bits), tiles in use
enum { LC_TILES = 0, LC_MASKS = TILE_REGIONS, LC_MAXHALF = 2*TILE_REGIONS, LC_USED = 2*TILE_REGIONS + 1, LC_STRIDE = 128 };

// indices into NbDev::counters
enum { CT_PAIRSTART = 0,      // SM partition: CTAs of the tile kernel that have started (see k_pair)
       CT_REBUILD = 2, CT_OVERFLOW = 3, CT_BUILDS = 4, CT_PAIRS = 5, CT_CUR = 10, CT_CURSOR = 14,
       CT_BTDONE = 7, CT_BAR = 9, CT_BAREXIT = 15 };      // k_build_tiles completion count; grid barrier of k_list_prep

struct NbDev {
    BoxDev box;
    int natoms, npad, nblocks;
    int method;                  // B200MD_NB_*
    int useSwitch;
    float cutoff, cutoff2, paddedCutoff2, switchDist;
    float alpha;                 // Ewald alpha
    float krf, crf;              // reaction field
    float dispDummy;
    // user-order state
    float4* posq;                // xyz + charge*sqrt(ONE_4PI_EPS0)
    float4* velm;                // v + 1/mass
    // mixed precision (b200md_set_precision): both null in a single-precision context.  Read and written only through the
    // state helpers below (load_pos / store_pos / vel_array); every force kernel keeps reading the fp32 posq.
    float4* posqCorr;            // low parts: position = posq.xyz + posqCorr.xyz (w unused)
    double4* velmD;              // v + 1/mass in double; replaces velm for every reader and writer
    float2* sigeps;             // (sigma/2, 2 sqrt(eps))  (ReferenceKernels.cpp:1093-1097)
    const double* chargeD;       // the same parameters in double (user order): the double-precision close-pair path
    const double2* sigepsD;
    long long* force;            // [3][npad] fixed point, user order
    // [3][npad] fixed point, sorted order of the current list: the tile kernel accumulates here (a warp's atomics land on
    // contiguous addresses), and k_fold_sorted, launched right behind it, adds it into `force` and zeroes it again
    long long* forceS;
    double* energy;              // [B200MD_NUM_ENERGY] accumulators
    // sorted (nonbonded) copies, blocks and tiles: two complete lists.  counters[CT_CUR] names the one the tile kernel reads;
    // a rebuild always fills the other one and flips at the end of k_build_tiles
    ListDev list[2];
    int* sortedOf;               // user atom -> sorted slot (of the list built last; list construction only)
    float4* refPos;              // user-order positions at the last list build
    // binning
    int ncell[3];
    int ncells;
    const int* cellRank;         // linear cell -> rank along the space filling curve
    int* cellCount;              // [ncells+1] -> after scan: start offsets
    int* cellFill;               // [ncells]
    int* atomCell;               // [natoms] rank of the atom's cell
    int* tmpSorted;              // [npad]
    float4* atomShift;           // [natoms]
    int maxTiles;
    int* counters;               // [2]=rebuild flag [3]=overflow [4]=list builds [5]=pairs(diag) [6]=nan flag
    // exclusions, CSR in user order
    const int* exclStart;
    const int* exclList;
    // whole molecules that have diffused more than one box length out of the primary cell are moved back by lattice vectors
    // at list builds (fp32 coordinates lose ~1e-7 nm of resolution per nm of magnitude: a water walks ~100 nm per
    // microsecond); cellOffset remembers the lattice vectors so that the user keeps seeing a continuous trajectory
    int nmol;                    // 0: wrapping off (non-periodic, or more than one rank)
    const int* molStart;         // CSR over molAtoms
    const int* molAtoms;
    int* cellOffset;             // [3][npad] lattice vector counts to ADD when reporting positions
    float halfPad2;              // (padding/2)^2: beyond this displacement the current list is invalid
    // multi-GPU sharding of the tile list / PME atoms
    int rank, world;
    // origin of the primary periodic cell used for binning (chosen at set_positions so that a structure centred anywhere,
    // e.g. a PDB centred on 0, is binned WITHOUT lattice shifts: a shift costs one fp32 rounding of the coordinate)
    double origin[3];
    // SM partition: the tile kernel's CTAs that land on an SM whose bit is set here return at once, so those SMs stay free for
    // the reciprocal-space chain (spread -> FFT -> gather) that runs beside it; the other CTAs (one persistent wave) share ALL
    // tiles through the cursor.  smPartition false (all bits zero): no partition, several waves, static tile stride.
    unsigned long long pmeSmMask[4];
    bool smPartition;
    float closeCut2;             // pairs closer than this (squared) are evaluated in double from the exact coordinates (0: off)
};

enum { EN_NB = 0, EN_RECIP = 1, EN_BOND = 2, EN_ANGLE = 3, EN_TORSION = 4, EN_EXC = 5, EN_KE = 6, EN_RBTORSION = 7, EN_CMAP = 8,
       EN_CUSTOM_TORSION = 9, B200MD_NUM_ENERGY = 10 };

struct PmeDev {
    int nx, ny, nz, nzc;
    real* grid;                  // real [nx][ny][nz] (output of the inverse transform, input of the gather)
    long long* gridFixed;        // real [nx][ny][nz], 2^32 fixed point: deterministic charge spreading (pme.cc:78-89 option)
    real2* cgrid;                // complex [nx][ny][nzc]
    real* eterm;                 // [nx][ny][nzc] influence function (no ONE_4PI_EPS0: charges carry sqrt of it)
    const double* moduli[3];
    FftPlanDev plan[3];          // x, y, z
    double alpha;
    // brick path of the spread (pme.cu): each CTA takes brickAtoms consecutive atoms of the current neighbour list's sorted
    // order and accumulates into a shared-memory box of at most brickPoints grid points.
    // brickAtoms == 0: user atom order, straight to global memory (multi-GPU, stand-alone PME, no list built yet)
    int brickAtoms;
    int brickPoints;
};

struct BondedDev {
    int nbonds, nangles, ntorsions, nrb, ncmap, nexc;
    const int2* bondAtoms; const double2* bondParams;           // (r0, k)
    const int4* angleAtoms; const double2* angleParams;         // (theta0, k)
    const int4* torsionAtoms; const double4* torsionParams;     // (k, phase, n, 0)
    const int4* rbAtoms; const double* rbParams;                // [nrb][6] Ryckaert-Bellemans c0..c5
    // CMAP: two dihedrals per term (atoms [2i], [2i+1]), a map index per term, per map (first patch, size), and the bicubic
    // coefficients of every patch, [sum size^2][16] (CMAPTorsionForceImpl::calcMapDerivatives), patch s + size*t of a map
    const int4* cmapAtoms; const int* cmapMap; const int2* cmapMaps; const double* cmapCoeff;
    const int2* excAtoms; const double4* excParams;             // (qq14*ONE_4PI_EPS0, sigma, 4 eps, 0)
    int excPeriodic;
    // force group of every bonded term (several Force objects of one class may sit in different groups,
    // ContextImpl::calcForcesAndEnergy groups, ContextImpl.cpp:293-308); an element is evaluated iff bit `group` of groupMask is set
    const unsigned char* bondGroup; const unsigned char* angleGroup; const unsigned char* torsionGroup;
    const unsigned char* rbGroup; const unsigned char* cmapGroup;
    unsigned int groupMask;
};

// Custom torsions (k_custom_torsion, bonded.cu): a kernel and a parameter block of their own, so that BondedDev and k_bonded
// stay as they are.  The terms are stored grouped by expression, each group padded to whole warps (prog = -1 in a padding
// slot), so that every warp runs one program and reads its code with uniform loads.  Program 2p is expression p's energy,
// program 2p+1 its dE/dtheta: the instructions [progStart[q], progStart[q+1]) of code (opcode, operand) and imm.
struct CustomTorsionDev {
    int nslots;                  // terms + padding
    int paramStride;             // parameters per slot
    const int4* atoms; const double* params; const unsigned char* group; const int* prog;
    const int2* code; const double* imm; const int* progStart;
    const double* globals;       // the values of the global parameter slots (b200md_set_custom_globals)
    unsigned int groupMask;
};

// One integration unit = a SETTLE water, a SHAKE cluster (centre + <=3 H) or a free atom.
struct UnitDev {
    int nunits;
    const int4* unitAtoms;       // atoms (unused = -1); SETTLE: (O,H1,H2,-1)
    const int* unitType;         // 0 free, 1 SETTLE, 2 SHAKE
    const float4* unitParams;    // SETTLE: (dOH, dHH, 0, 0); SHAKE: (d1, d2, d3, 0)
    const double4* unitParamsD;  // the same in double (mixed precision only)
};

struct IntegDev {
    int kind;
    float dt, vscale, fscale, noisescale;   // Langevin constants (ReferenceStochasticDynamics.cpp:94-99)
    float kT;
    float tol;
    double dtD, vscaleD, fscaleD, noisescaleD, kTD, tolD;   // the same in double (read by the mixed-precision kernels only)
    unsigned int seed;
    unsigned long long stepIndex;            // not used on device when graphs are active: see stepCounter
    unsigned long long* stepCounter;         // device counter, incremented by the integrate kernel
    int fused;                               // step path: zero forces, fused CM removal, last block advances the counter
    int cmEveryStep;                         // CMMotionRemover with frequency 1
    double* cmScratch;                       // [3][4] rotating momentum/mass accumulators
    unsigned int* blocksDone;
};

// ---------------------------------------------------------------------------------------------------------------
// Multi-GPU data plane (one process per GPU): every rank maps every other rank's WINDOW (one cudaMalloc, exported with
// cudaIpcGetMemHandle) and the kernels themselves move the data with plain stores over NVLink, tile by tile, and
// publish a flag per (channel, source rank) when a stage is complete; consumers spin on their LOCAL flag copy.  No
// NCCL call on the step path.  Ownership: rank q owns the user atoms [atomLo[q], atomLo[q+1]) (cut at integration-unit
// boundaries): it reduces their forces, integrates them and pushes their new positions to everybody.  Reciprocal space
// is slab-decomposed: rank q owns the x planes [xLo[q], xLo[q+1]) for the (y,z) transforms and the (ky,kz) lines
// [q*lineChunk, ...) for the x transform; the two transposes are the stores of the FFT kernels themselves.
#define B200MD_MAX_RANKS 8
enum { CH_POS = 0,      // new positions of the owner's atoms are in everybody's posq        (k_integrate)
       CH_FORCE = 1,    // partial forces are in the owners' inboxes                         (k_force_push)
       CH_FINAL = 2,    // total forces of the owner's atoms are in everybody's force buffer (k_force_total; compute path only)
       CH_GRID = 3,     // charge-grid contributions are in the slab owners' inboxes         (k_grid_push)
       CH_FWD = 4,      // (y,z)-transformed planes are in the line owners' buffers          (k_fft_slab_fwd)
       CH_INV = 5,      // x-transformed, convolved lines are back in the slab owners' buffers (k_fft_x_conv)
       CH_POT = 6,      // potential planes are in everybody's grid                          (k_fft_slab_inv)
       CH_VEL = 7,      // velocities of the owner's atoms are in everybody's velm           (k_vel_push; state reads only)
       CH_COUNT = 8 };
struct CommDev {
    int rank, world;                     // world == 1: no peer traffic, every wait/signal is skipped
    int atomLo[B200MD_MAX_RANKS + 1];
    int unitLo[B200MD_MAX_RANKS + 1];
    int xLo[B200MD_MAX_RANKS + 1];       // x planes of the PME grid
    int lineChunk;                       // (ky,kz) lines per rank (multiple of the x-pass batch; the last rank may get fewer)
    int maxPlanes;                       // max x planes per rank
    char* peer[B200MD_MAX_RANKS];        // window base of every rank as mapped HERE (peer[rank] = own window)
    // offsets inside a window (identical on every rank)
    size_t offFlags, offPosq, offVelm, offForce, offFinbox, offCm, offGridInbox, offLineBuf, offPlaneBuf, offGrid;
    unsigned long long* epoch;           // local: number of completed exchanges; every evaluation uses E = *epoch + 1
    unsigned long long* posNeed;         // local: CH_POS value the next evaluation must wait for (0: positions were set by the host)
    unsigned int* done;                  // local: [CH_COUNT] block-completion counters of the signalling kernels
    int* errFlag;                        // local: sticky error (NbDev::counters + CT_OVERFLOW): a wait that times out raises 3
    int posByPush;                       // 1: k_integrate writes positions locally only, k_pos_push (TMA) publishes them and CH_POS
};

#ifdef __CUDACC__
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long* comm_flag(const CommDev& cd, int onRank, int ch, int src) {
    return (unsigned long long*) (cd.peer[onRank] + cd.offFlags) + ch*B200MD_MAX_RANKS + src;
}
// Block-wide: wait until every peer has published `need` on channel ch.  Bounded (~1 s): a lost peer raises the sticky
// error flag instead of hanging the device.
__device__ __forceinline__ void comm_wait(const CommDev& cd, int ch, unsigned long long need) {
    if (cd.world > 1 && need != 0ull) {
        if (threadIdx.x < cd.world && (int) threadIdx.x != cd.rank && threadIdx.y == 0 && threadIdx.z == 0) {
            const unsigned long long* f = comm_flag(cd, cd.rank, ch, threadIdx.x);
            long spins = 0;
            while (ld_acquire_sys(f) < need) {
                if (*((volatile int*) cd.errFlag) == 3) break;        // a peer was lost earlier: fail fast, the host raises at its next sync
                __nanosleep(64);
                if (++spins > (1L << 22)) { *cd.errFlag = 3; break; }
            }
        }
    }
    __syncthreads();
}
// Block-wide: this block's stores to peer memory are complete.  Returns true (to all threads) in the LAST block of the grid,
// which then publishes the stage with comm_publish (possibly after a little more work of its own).
__device__ __forceinline__ bool comm_arrive(const CommDev& cd, int ch, unsigned int nblocks) {
    __shared__ int lastBlock;
    __syncthreads();                   // the block's stores happen-before thread 0's fence (cumulativity): ONE system fence per CTA
    if (threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0) {
        __threadfence_system();
        lastBlock = (atomicAdd(&cd.done[ch], 1u) == nblocks - 1u);
        if (lastBlock) { cd.done[ch] = 0u; __threadfence_system(); }
    }
    __syncthreads();
    return lastBlock != 0;
}
__device__ __forceinline__ void comm_publish(const CommDev& cd, int ch, unsigned long long value) {       // one thread
    __threadfence_system();
    for (int k = 1; k < cd.world; k++) { const int q = (cd.rank + k) % cd.world; st_release_sys(comm_flag(cd, q, ch, cd.rank), value); }
}
__device__ __forceinline__ bool comm_signal(const CommDev& cd, int ch, unsigned long long value, unsigned int nblocks) {
    const bool last = comm_arrive(cd, ch, nblocks);
    if (last && threadIdx.x == 0 && threadIdx.y == 0 && threadIdx.z == 0) comm_publish(cd, ch, value);
    return last;
}
__device__ __forceinline__ int comm_owner_of_atom(const CommDev& cd, int a) {
    int q = 0;
#pragma unroll
    for (int k = 1; k < B200MD_MAX_RANKS; k++) q += (k < cd.world && a >= cd.atomLo[k]) ? 1 : 0;
    return q;
}
#endif

// 2^32 fixed point <-> fp32 without the 64-bit conversion instructions (I2F.S64 / F2I.S64 are multi-pass on the XU pipe and
// showed up as the hottest instructions of the FFT load loop and of the integrator in the round-1 profiles)
#ifdef __CUDACC__
__device__ __forceinline__ float fixed_to_float(long long v) {
    const int hi = (int) (v >> 32);
    const unsigned int lo = (unsigned int) v;
    return __int2float_rn(hi) + __uint2float_rn(lo)*2.3283064365386963e-10f;
}
__device__ __forceinline__ long long float_to_fixed(float f) {           // |f| < 2^31
    const float fl = floorf(f);
    const int hi = __float2int_rd(f);
    const unsigned int lo = __float2uint_rz((f - fl)*4294967296.0f);
    return ((long long) hi << 32) | (long long) lo;
}

// ---- integration state in the working type R: float (single precision) or double (mixed precision) ----
// The only place that knows the mixed layout: a position is posq.xyz (hi) + posqCorr.xyz (lo), stored as hi = (float) x,
// lo = (float) (x - hi), about 48 significant bits; velocities and 1/mass live in velmD.  The fp32 posq the force kernels
// read is the hi part, so forces at a given posq do not depend on the precision.
__host__ __device__ __forceinline__ void pos_split(double x, float& hi, float& lo) { hi = (float) x; lo = (float) (x - (double) hi); }
__host__ __device__ __forceinline__ double pos_join(float hi, float lo) { return (double) hi + (double) lo; }
template <class R> struct Vec4Of;
template <> struct Vec4Of<float> { typedef float4 T; };
template <> struct Vec4Of<double> { typedef double4 T; };
template <class R> using R4 = typename Vec4Of<R>::T;

__device__ __forceinline__ float4 make_r4(float x, float y, float z, float w) { return make_float4(x, y, z, w); }
__device__ __forceinline__ double4 make_r4(double x, double y, double z, double w) { return make_double4(x, y, z, w); }

// position (xyz) and charge (w)
template <class R> __device__ R4<R> load_pos(const NbDev& nb, int a);
template <> __device__ __forceinline__ float4 load_pos<float>(const NbDev& nb, int a) { return nb.posq[a]; }
template <> __device__ __forceinline__ double4 load_pos<double>(const NbDev& nb, int a) {
    const float4 h = nb.posq[a], l = nb.posqCorr[a];
    return make_double4(pos_join(h.x, l.x), pos_join(h.y, l.y), pos_join(h.z, l.z), (double) h.w);
}
// new position of atom a; the charge in posq.w is kept
template <class R> __device__ void store_pos(const NbDev& nb, int a, R x, R y, R z);
template <> __device__ __forceinline__ void store_pos<float>(const NbDev& nb, int a, float x, float y, float z) {
    nb.posq[a] = make_float4(x, y, z, nb.posq[a].w);
}
template <> __device__ __forceinline__ void store_pos<double>(const NbDev& nb, int a, double x, double y, double z) {
    float hx, hy, hz, lx, ly, lz;
    pos_split(x, hx, lx); pos_split(y, hy, ly); pos_split(z, hz, lz);
    nb.posq[a] = make_float4(hx, hy, hz, nb.posq[a].w);
    nb.posqCorr[a] = make_float4(lx, ly, lz, 0.f);
}
// velocities + 1/mass (w)
template <class R> __device__ R4<R>* vel_array(const NbDev& nb);
template <> __device__ __forceinline__ float4* vel_array<float>(const NbDev& nb) { return nb.velm; }
template <> __device__ __forceinline__ double4* vel_array<double>(const NbDev& nb) { return nb.velmD; }

template <class R> __device__ R fixed_to_real(long long v);
template <> __device__ __forceinline__ float fixed_to_real<float>(long long v) { return fixed_to_float(v); }
template <> __device__ __forceinline__ double fixed_to_real<double>(long long v) { return (double) v*(1.0/B200MD_FORCE_SCALE); }

__device__ __forceinline__ float rsqrt_r(float x) { return rsqrtf(x); }
__device__ __forceinline__ double rsqrt_r(double x) { return rsqrt(x); }
__device__ __forceinline__ float sqrt_r(float x) { return sqrtf(x); }
__device__ __forceinline__ double sqrt_r(double x) { return sqrt(x); }
__device__ __forceinline__ float fabs_r(float x) { return fabsf(x); }
__device__ __forceinline__ double fabs_r(double x) { return fabs(x); }
#endif

// integrator constants in the working type (IntegDev keeps both: fp32 for single precision, double for mixed)
template <class R> struct IntegR { R dt, vscale, fscale, noisescale, kT, tol; };
#ifdef __CUDACC__
template <class R> __device__ IntegR<R> integ_r(const IntegDev& in);
template <> __device__ __forceinline__ IntegR<float> integ_r<float>(const IntegDev& in) { return {in.dt, in.vscale, in.fscale, in.noisescale, in.kT, in.tol}; }
template <> __device__ __forceinline__ IntegR<double> integ_r<double>(const IntegDev& in) { return {in.dtD, in.vscaleD, in.fscaleD, in.noisescaleD, in.kTD, in.tolD}; }
#endif

// General constraint networks (CCMA, constraints.cu): one CTA per connected component of the constraint graph.
struct CcmaDev {
    int ncomp, ncon, natomsC;
    const int* compConStart;     // [ncomp+1] constraints of a component are contiguous
    const int* compAtomStart;    // [ncomp+1] so are its atoms (positions in `atoms`)
    const int2* conAtoms;        // [ncon] user atom indices
    const float* conDist;        // [ncon]
    const float* conRedMass;     // [ncon] 0.5/(1/mi + 1/mj)
    const int* rowStart; const int* col; const float* val;      // approximate inverse of the coupling matrix, CSR over constraints
    const int* atoms;            // [natomsC] user atom index
    const int* aStart;           // [natomsC+1] constraints of an atom: +(k+1) if it is the first atom of constraint k, -(k+1) if the second
    const int* aCon;
    float4* rij; float* delta1; float* delta2;                   // [ncon] scratch
    float4* xold; float4* xunc;                                  // [npad] scratch (user atom order)
    int maxIter;
    // mixed precision only: constants and scratch in double; xpos holds the positions the solver works on (hi + lo)
    const double* conDistD; const double* conRedMassD;
    double4* rijD; double* delta1D; double* delta2D;
    double4* xoldD; double4* xuncD; double4* xposD;
};

#ifdef __CUDACC__
// ---------------------------------------------------------------- Philox4x32-10 (Salmon et al., SC'11)
__device__ __forceinline__ uint4 philox(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; r++) {
        const unsigned int hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u*c.x;
        const unsigned int hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u*c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u; k.y += 0xBB67AE85u;
    }
    return c;
}

// three independent N(0,1) for (atom, step)
__device__ __forceinline__ float3 gauss3(unsigned int seed, int atom, unsigned long long step) {
    uint4 r = philox(make_uint4((unsigned int) atom, (unsigned int) step, (unsigned int) (step >> 32), 0x5eed5eedu), make_uint2(seed, 0xb200b200u));
    const float u1 = ((r.x >> 8) + 1u)*(1.0f/16777216.0f);      // (0,1]
    const float u2 = (r.y >> 8)*(1.0f/16777216.0f);
    const float u3 = ((r.z >> 8) + 1u)*(1.0f/16777216.0f);
    const float u4 = (r.w >> 8)*(1.0f/16777216.0f);
    const float m1 = sqrtf(-2.0f*logf(u1)), m2 = sqrtf(-2.0f*logf(u3));
    float s1, c1, s2, c2;
    sincospif(2.0f*u2, &s1, &c1);
    sincospif(2.0f*u4, &s2, &c2);
    (void) s2;
    return make_float3(m1*c1, m1*s1, m2*c2);
}

#endif

// Monte Carlo barostat move (k_scale_molecules): molecules as ContextImpl::getMolecules() forms them, the current box vectors in
// double (reduced form, a = (a0,0,0), b = (b0,b1,0)) and the scale factor of each axis.
struct ScaleDev {
    int nmol;
    const int* molStart;         // [nmol+1] CSR over molAtoms
    const int* molAtoms;
    double a[3], b[3], c[3];
    double s[3];
};

// ---- launchers (defined in the .cu files) ----
void launch_check_displacement(const NbDev& nb, const CommDev& cd, cudaStream_t s);
const int LIST_BUILD_LAUNCHES = 2;
void launch_list_build(const NbDev& nb, cudaStream_t s);     // k_list_prep (grid barriers) + k_build_tiles, gated on counters[CT_REBUILD]
const int PAIR_LAUNCHES = 2;
void launch_pair(const NbDev& nb, bool energy, cudaStream_t s);        // k_pair + k_fold_sorted (sorted -> user-order forces)
void pair_set_carveout(size_t fftSmem, size_t brickSmem);     // shared memory for a chain CTA beside the tile CTAs left on an SM
void launch_count_pairs(const NbDev& nb, cudaStream_t s);
int choose_pme_sms(int reserve, unsigned long long mask[4]);     // SM partition of the tile kernel (NbDev::pmeSmMask)

void launch_pme_eterm(const NbDev& nb, const PmeDev& pme, cudaStream_t s);
// zeroGrid = false: the caller has zeroed pme.gridFixed on this stream already (the single-GPU step does it at its head)
void launch_pme_spread(const NbDev& nb, const PmeDev& pme, const CommDev& cd, cudaStream_t s, bool zeroGrid = true);
// besideTiles: one GPU, the chain shares every SM with the tile kernel (smaller FFT CTAs, fft.cu)
void launch_pme_fft_conv(const NbDev& nb, const PmeDev& pme, const CommDev& cd, bool energy, bool besideTiles, cudaStream_t s);
void launch_pme_gather(const NbDev& nb, const PmeDev& pme, const CommDev& cd, cudaStream_t s);
void pme_brick_setup(int maxSmem);
void launch_grid_push(const PmeDev& pme, const CommDev& cd, cudaStream_t s);
void launch_fft3d_r2c(const PmeDev& pme, cudaStream_t s);         // grid -> cgrid
void launch_fft3d_c2r(const PmeDev& pme, cudaStream_t s);         // cgrid -> grid
size_t fft_plane_smem_bytes(int ny, int nz);
size_t fft_line_smem_bytes(int nx);
bool fft_make_radices(int n, int* radix, int* nstages);
int pme_fft_launch_count(const PmeDev& pme);
void fft_set_compact(int on);                   // smaller FFT CTAs (the chain shares the GPU with the tile kernel)
size_t fft_cta_smem_bytes(const PmeDev& pme);  // largest shared memory of one single-GPU FFT CTA of this grid (dynamic + static)
bool fft_slab_path(const PmeDev& pme);          // the 3-launch slab pipeline is usable for this grid (precondition of the multi-GPU FFT)

// k_bonded (when the classes in `terms` have terms) and, when `terms` has B200MD_TERM_CUSTOM_TORSIONS and there are custom
// torsions, k_custom_torsion behind it on the same stream
void launch_bonded(const NbDev& nb, const BondedDev& bd, const CustomTorsionDev& ct, int terms, bool energy, cudaStream_t s);
void launch_custom_torsion(const NbDev& nb, const CustomTorsionDev& ct, bool energy, cudaStream_t s);

void launch_integrate(const NbDev& nb, const UnitDev& units, const IntegDev& integ, const CommDev& cd, cudaStream_t s);
void launch_force_push(const NbDev& nb, const CommDev& cd, cudaStream_t s);          // partial forces of foreign atoms -> owners' inboxes
void launch_pos_push(const NbDev& nb, const CommDev& cd, const IntegDev& in, cudaStream_t s);   // owned positions -> every peer (TMA); publishes CH_POS
bool pos_push_available();
void launch_force_total(const NbDev& nb, const CommDev& cd, cudaStream_t s);         // compute path: owners total and broadcast, everybody waits
void launch_vel_push(const NbDev& nb, const CommDev& cd, cudaStream_t s);            // owners' velocities -> everybody (state reads)
void launch_pos_wait(const NbDev& nb, const CommDev& cd, cudaStream_t s);            // wait for the peers' position stores (state reads)
// every launcher below runs the double (mixed-precision) instantiation when nb.velmD is set; tolerances and time shifts arrive
// in double and the single-precision kernels round them to fp32
void launch_constrain_positions(const NbDev& nb, const UnitDev& units, double tol, cudaStream_t s);
void launch_constrain_velocities(const NbDev& nb, const UnitDev& units, double tol, cudaStream_t s);
void launch_kinetic_energy(const NbDev& nb, const UnitDev& units, const IntegDev& integ, double shiftDt, cudaStream_t s);
void launch_remove_cm(const NbDev& nb, double* scratch, cudaStream_t s);
void launch_scale_molecules(const NbDev& nb, const ScaleDev& sc, cudaStream_t s);
void launch_ccma_step(const NbDev& nb, const CcmaDev& cc, const IntegDev& in, cudaStream_t s);      // before launch_integrate in a step
void launch_ccma_apply(const NbDev& nb, const CcmaDev& cc, bool velocities, double tol, cudaStream_t s);
void launch_ccma_kinetic(const NbDev& nb, const CcmaDev& cc, double shiftDt, double tol, cudaStream_t s);
void launch_cm_prime(const NbDev& nb, const IntegDev& integ, const CommDev& cd, cudaStream_t s);
