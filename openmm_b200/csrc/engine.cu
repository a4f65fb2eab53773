// engine.cu -- host side of libb200md.so: the C-ABI of include/b200md.h over the CUDA kernels of this directory.
// No CPU fallback exists: every compute entry point needs a CUDA device and fails loudly without one.
#include "engine.h"
#include "custom_interp.h"
#include "../../include/b200md.h"
#include <stdexcept>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <map>
#include <set>
#include <dlfcn.h>
#include <thread>

static std::string g_create_error;

template <class T> struct DevBuf {
    T* p = nullptr; size_t n = 0; bool owned = true;
    // attach: the buffer lives inside the multi-GPU window (peers store into it); alloc() then only checks the size
    void attach(void* ptr, size_t count) { free(); p = (T*) ptr; n = count; owned = false; }
    void alloc(size_t count) {
        if (!owned) { if (count > n) throw std::runtime_error("window buffer too small"); return; }
        free(); n = count; if (count) CUDA_CHECK(cudaMalloc(&p, count*sizeof(T)));
    }
    void upload(const std::vector<T>& v) { if (v.size() > n) alloc(v.size()); if (!v.empty()) CUDA_CHECK(cudaMemcpy(p, v.data(), v.size()*sizeof(T), cudaMemcpyHostToDevice)); }
    void zero() { if (n) CUDA_CHECK(cudaMemset(p, 0, n*sizeof(T))); }
    void free() { if (p && owned) cudaFree(p); p = nullptr; n = 0; owned = true; }
    ~DevBuf() { free(); }
};

static void require(bool cond, const char* msg) { if (!cond) throw std::runtime_error(msg); }

// A device-side copy of some of the context's arrays (`parts`), packed into one buffer.
struct DevSpan { void* p; size_t bytes; };
struct Snapshot {
    std::vector<DevSpan> parts;
    DevBuf<char> buf;
    void save(cudaStream_t s) {
        size_t total = 0;
        for (const DevSpan& q : parts) total += q.bytes;
        if (buf.n != total) buf.alloc(total);
        char* d = buf.p;
        for (const DevSpan& q : parts) { CUDA_CHECK(cudaMemcpyAsync(d, q.p, q.bytes, cudaMemcpyDeviceToDevice, s)); d += q.bytes; }
    }
    void restore(cudaStream_t s) const {
        const char* d = buf.p;
        for (const DevSpan& q : parts) { CUDA_CHECK(cudaMemcpyAsync(q.p, d, q.bytes, cudaMemcpyDeviceToDevice, s)); d += q.bytes; }
    }
};

// Every atom index of a packed term table lies in [0, natoms): every int component, the 0 that pads an angle's int4 included.
template <class A> static void check_atoms(int natoms, const std::vector<A>& a, const char* cls) {
    const int* q = (const int*) a.data();
    for (size_t k = 0; k < a.size()*sizeof(A)/sizeof(int); k++)
        if (q[k] < 0 || q[k] >= natoms) throw std::runtime_error(std::string(cls) + ": atom index out of range");
}

// One bonded term class in the layout BondedDev reads: n terms' atoms and parameters, each term's force group (none set =
// group 0) and the device copies.  set_* fills it through set(), finalize uploads it, update_* rewrites `params` and uploads
// them into the same buffers (same size: captured step graphs keep their pointers).
template <class A, class P> struct TermTable {
    int n = 0;
    std::vector<A> atoms; std::vector<P> params; std::vector<unsigned char> group;
    DevBuf<A> atomsDev; DevBuf<P> paramsDev; DevBuf<unsigned char> groupDev;
    void set(int natoms, const char* cls, int count, std::vector<A>& a, std::vector<P>& p) {
        check_atoms(natoms, a, cls);
        n = count; atoms.swap(a); params.swap(p);
    }
    // finalize: upload, and point the BondedDev fields at the copies (groups may come before or after the terms)
    void upload(int& count, const A*& a, const P*& p, const unsigned char*& g) {
        require(group.empty() || (int) group.size() == n, "set_bonded_groups: group array length differs from the number of terms");
        std::vector<unsigned char> gr(group); gr.resize(std::max(n, 1), 0);
        atomsDev.upload(atoms); paramsDev.upload(params); groupDev.upload(gr);
        count = n; a = atomsDev.p; p = paramsDev.p; g = groupDev.p;
    }
};
// CMAP: two int4 (the two dihedrals) per term, params = the coefficients of every patch [sum size^2][16]; besides, the map
// index of every term and per map (first patch, size)
struct CmapTable : TermTable<int4, double> {
    std::vector<int> map; std::vector<int2> maps;
    DevBuf<int> mapDev; DevBuf<int2> mapsDev;
};
// Custom torsions: atoms, params [n][stride] and groups in the caller's term order; besides, the programs (code = (opcode,
// operand), imm, progStart), the expression of every term and the global values.  finalize lays the terms out as
// k_custom_torsion reads them: grouped by expression, each group padded to whole warps; slot[i] is the slot of term i.
struct CustomTorsionTable : TermTable<int4, double> {
    int stride = 0, nprog = 0, nslots = 0;
    std::vector<int2> code; std::vector<double> imm; std::vector<int> progStart, prog, slot;
    std::vector<double> globals;
    DevBuf<int2> codeDev; DevBuf<double> immDev, globalsDev; DevBuf<int> progStartDev, progDev;
    // params in the slot layout (padding slots 0)
    std::vector<double> slot_params() const {
        std::vector<double> p((size_t) nslots*stride, 0.0);
        for (int i = 0; i < n; i++) std::copy(params.begin() + (size_t) i*stride, params.begin() + (size_t) (i+1)*stride, p.begin() + (size_t) slot[i]*stride);
        return p;
    }
};

// The buffers of one neighbour list (ListDev): the sorted copies and the block boxes, sized by the atoms; the tile pools,
// sized by the tile capacity and grown by prepare_list.
struct ListBufs {
    DevBuf<float4> sposq, swrap, blockCenter, blockHalf, superCenter, superHalf;
    DevBuf<float2> ssigeps; DevBuf<double> schargeD; DevBuf<double2> ssigepsD;
    DevBuf<int> sorig, tileI, tileJ, tileMask; DevBuf<unsigned int> maskPool;
    void alloc(int npad, int nblocks) {
        sposq.alloc(npad); sposq.zero(); swrap.alloc(npad); swrap.zero(); ssigeps.alloc(npad); ssigeps.zero();
        sorig.alloc(npad); sorig.zero(); blockCenter.alloc(nblocks); blockHalf.alloc(nblocks);
        schargeD.alloc(npad); schargeD.zero(); ssigepsD.alloc(npad); ssigepsD.zero();
        superCenter.alloc((nblocks + 31)/32); superHalf.alloc((nblocks + 31)/32);
    }
    void alloc_tiles(int maxTiles) {
        tileI.alloc(maxTiles); tileJ.alloc((size_t) maxTiles*32); tileMask.alloc(maxTiles); maskPool.alloc((size_t) maxTiles*32);
    }
    void bind(ListDev& L, int* lc) const {
        L.sposq = sposq.p; L.ssigeps = ssigeps.p; L.schargeD = schargeD.p; L.ssigepsD = ssigepsD.p; L.swrap = swrap.p; L.sorig = sorig.p;
        L.blockCenter = blockCenter.p; L.blockHalf = blockHalf.p; L.superCenter = superCenter.p; L.superHalf = superHalf.p;
        L.tileI = tileI.p; L.tileJ = tileJ.p; L.tileMask = tileMask.p; L.maskPool = maskPool.p; L.lc = lc;
    }
};

// ---- minimal NCCL binding, resolved at run time so that libb200md.so has no link-time NCCL dependency ----
struct NcclUid { char b[128]; };      // ncclUniqueId is passed BY VALUE to ncclCommInitRank
struct NcclApi {
    typedef NcclUid Uid;
    void* lib = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(void**, int, NcclUid, int) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, void*, cudaStream_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load(std::string& err) {
        if (lib) return true;
        const char* names[] = {getenv("B200MD_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) { if (nm && (lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL))) break; }
        if (!lib) { err = "cannot dlopen libnccl (set B200MD_NCCL_LIB)"; return false; }
        GetUniqueId = (decltype(GetUniqueId)) dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank)) dlsym(lib, "ncclCommInitRank");
        AllReduce = (decltype(AllReduce)) dlsym(lib, "ncclAllReduce");
        AllGather = (decltype(AllGather)) dlsym(lib, "ncclAllGather");
        CommDestroy = (decltype(CommDestroy)) dlsym(lib, "ncclCommDestroy");
        GetErrorString = (decltype(GetErrorString)) dlsym(lib, "ncclGetErrorString");
        if (!GetUniqueId || !CommInitRank || !AllReduce) { err = "libnccl lacks required symbols"; return false; }
        return true;
    }
};
static NcclApi g_nccl;
enum { NCCL_INT8 = 0, NCCL_INT64 = 4, NCCL_FLOAT32 = 7, NCCL_FLOAT64 = 8, NCCL_SUM = 0 };

struct b200md_ctx {
    int device = 0;
    int natoms = 0, npad = 0, nblocks = 0;
    bool finalized = false;
    std::string err;
    cudaStream_t stream = nullptr;
    cudaStream_t streamPme = nullptr;   // reciprocal space runs concurrently with direct space (high priority: its kernels are small)
    cudaStream_t streamBonded = nullptr;    // one GPU: the bonded terms, beside both
    cudaEvent_t evFork = nullptr, evJoin = nullptr, evJoinBonded = nullptr, evForkGrid = nullptr;
    bool pmeOnly = false;               // b200md_pme_create: reciprocal space only, no neighbour list is ever built
    bool listDirty = true;              // state changed from outside: rebuild synchronously before the next step graph
    bool overlapPme = true;
    // brick path of the PME spread (pme.cu): B200MD_PME_BRICK=0 keeps the user-order kernel; B200MD_PME_BRICK_POINTS sets
    // the brick capacity (a small one forces the global-memory fallback)
    bool pmeBrick = true;
    int brickAtoms = 64, brickPoints = 8192;
    bool listBuilt = false;             // a neighbour list covers every atom (the brick path walks its sorted order)
    // ---- host copy of the system definition ----
    std::vector<double> mass, charge, sigma, epsilon;
    b200md_nonbonded_desc nbdesc{};
    bool haveNb = false;
    // exceptions keep (qq, sigma, eps) as given: the device double4 also holds the product of the charges (upload_params)
    struct { std::vector<int2> atoms; std::vector<double3> params; DevBuf<int2> atomsDev; DevBuf<double4> paramsDev; } exc;
    TermTable<int2, double2> bonds;         // (r0, k)
    TermTable<int4, double2> angles;        // atoms (i, j, k, 0), (theta0, k)
    TermTable<int4, double4> torsions;      // (k, phase, n, 0)
    TermTable<int4, double> rb;             // [n][6] c0..c5
    CmapTable cmap;
    CustomTorsionTable custom;
    std::vector<int> conI, conJ; std::vector<double> conD;
    int cmFreq = 0;
    std::vector<int4> hUnitAtoms;        // host copy of the integration units (ownership cuts of the multi-GPU data plane)
    double boxA[3] = {0, 0, 0}, boxB[3] = {0, 0, 0}, boxC[3] = {0, 0, 0};
    bool haveBox = false;
    bool haveOrigin = false;
    double padFrac = 0.10;
    // ---- device state ----
    DevBuf<float4> posq, velm, refPos, atomShift;
    DevBuf<float2> sigeps;
    DevBuf<double> chargeD; DevBuf<double2> sigepsD;
    ListBufs lists[2];
    DevBuf<long long> force, forceS;
    DevBuf<double> energy, cmScratch;
    DevBuf<int> molStart, molAtoms, cellOffset, sortedOf, cellRank, cellCount, cellFill, atomCell, tmpSorted, listCounters, counters, exclStart, exclList;
    DevBuf<unsigned long long> stepCounter;
    DevBuf<unsigned int> blocksDone;
    bool stepStateValid = false;         // fused step path: force buffer zeroed and cm accumulator primed
    DevBuf<real> grid, eterm;
    DevBuf<long long> gridFixed;
    DevBuf<real2> cgrid;
    DevBuf<real2> tw[3];
    DevBuf<double> moduli[3];
    DevBuf<int4> unitAtoms; DevBuf<int> unitType; DevBuf<float4> unitParams;
    // general constraint networks (CCMA, constraints.cu)
    std::vector<int> ccmaCons;           // indices into conI/conJ/conD
    DevBuf<int> ccCompCon, ccCompAtom, ccRowStart, ccCol, ccAtoms, ccAStart, ccACon;
    DevBuf<int2> ccConAtoms; DevBuf<float> ccDist, ccRedMass, ccVal, ccDelta1, ccDelta2;
    DevBuf<float4> ccRij, ccXold, ccXunc;
    // mixed precision (b200md_set_precision): low parts of the positions, double velocities, double constraint constants and
    // CCMA scratch; unallocated in a single-precision context
    int precision = B200MD_PRECISION_SINGLE;
    DevBuf<float4> posqCorr; DevBuf<double4> velmD, unitParamsD;
    DevBuf<double> ccDistD, ccRedMassD, ccDelta1D, ccDelta2D; DevBuf<double4> ccRijD, ccXoldD, ccXuncD, ccXposD;
    bool mixed() const { return precision == B200MD_PRECISION_MIXED; }
    CcmaDev ccma{};
    NbDev nb{};
    PmeDev pme{};
    BondedDev bd{};
    CustomTorsionDev ctd{};
    UnitDev units{};
    IntegDev integ{};
    bool haveIntegrator = false;
    double dt = 0, temperature = 0, friction = 0;
    double time = 0;
    int64_t stepCount = 0;
    double selfEnergy = 0, dispersionCoefficient = 0;
    // ---- stats ----
    int64_t forceEvals = 0, kernelLaunches = 0, graphInstantiations = 0;
    // ---- Monte Carlo barostat (b200md_scale_coordinates / b200md_restore_coordinates) ----
    DevBuf<int> baroStart, baroAtoms;    // molecules of ContextImpl::getMolecules(), CSR
    int baroNmol = 0;
    Snapshot baroSave;                   // positions, cellOffset and forces before the last scale (no parts: no scale yet)
    // ---- graph ----
    cudaGraphExec_t stepGraph = nullptr;      // one MD step
    cudaGraphExec_t multiGraph = nullptr;     // graphSteps MD steps in one launch (host launch cost amortised)
    bool graphValid = false;                  // stepGraph matches the current kernel parameters
    bool multiValid = false;                  // multiGraph does
    bool useGraph = true;
    int graphSteps = 8;
    int stepLaunches = 0;
    // ---- multi-GPU ----
    void* comm = nullptr;
    int rank = 0, world = 1;
    // peer-memory data plane (comm.cu): one window per rank, mapped by every other rank with CUDA IPC
    bool p2p = false;                    // world > 1 and B200MD_MGPU != nccl
    CommDev cd{};                        // world == 1 unless p2p
    char* window = nullptr; size_t windowBytes = 0;
    void* peerMapped[B200MD_MAX_RANKS] = {nullptr};
    DevBuf<unsigned long long> commCounters;   // [0] epoch, [1] posNeed
    DevBuf<unsigned int> commDone;             // [CH_COUNT]
    bool velStale = false;               // p2p: the velocities of foreign atoms are behind (only owners integrate)
    std::vector<float4> hbuf4, hcorr4;
    std::vector<int> hoffset;
    std::vector<long long> hforce;
};

#define API_BEGIN(ctx) if (!(ctx)) return -1; try { CUDA_CHECK(cudaSetDevice((ctx)->device));
#define API_END(ctx) } catch (std::exception& e) { (ctx)->err = e.what(); return -1; } return 0;

static void check_flags(b200md_ctx* c);
static void sync_velocities(b200md_ctx* c);
static void sync_positions(b200md_ctx* c);

extern "C" const char* b200md_version(void) { return "b200md 0.2 (sm_90a)"; }
extern "C" const char* b200md_last_error(const b200md_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_error.c_str(); }

extern "C" int b200md_create(b200md_ctx** out, int device, int natoms) {
    try {
        require(out != nullptr && natoms > 0, "b200md_create: bad arguments");
        int count = 0;
        cudaError_t e = cudaGetDeviceCount(&count);
        if (e != cudaSuccess || count == 0)
            throw std::runtime_error(std::string("b200md_create: no CUDA device available (") + cudaGetErrorString(e) + "); this library has no CPU fallback");
        require(device >= 0 && device < count, "b200md_create: device index out of range");
        CUDA_CHECK(cudaSetDevice(device));
        b200md_ctx* c = new b200md_ctx();
        c->device = device;
        c->natoms = natoms;
        c->npad = ((natoms + 31)/32)*32;
        c->nblocks = c->npad/32;
        CUDA_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
        if (getenv("B200MD_NO_OVERLAP")) c->overlapPme = false;
        if (getenv("B200MD_PME_BRICK")) c->pmeBrick = atoi(getenv("B200MD_PME_BRICK")) != 0;
        if (getenv("B200MD_PME_BRICK_POINTS")) c->brickPoints = std::max(1, atoi(getenv("B200MD_PME_BRICK_POINTS")));
        int hi = 0;
        CUDA_CHECK(cudaDeviceGetStreamPriorityRange(nullptr, &hi));
        CUDA_CHECK(cudaStreamCreateWithPriority(&c->streamPme, cudaStreamNonBlocking, hi));
        CUDA_CHECK(cudaStreamCreateWithPriority(&c->streamBonded, cudaStreamNonBlocking, hi));
        CUDA_CHECK(cudaEventCreateWithFlags(&c->evFork, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&c->evJoin, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&c->evJoinBonded, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&c->evForkGrid, cudaEventDisableTiming));
        c->mass.assign(natoms, 1.0);
        c->charge.assign(natoms, 0.0); c->sigma.assign(natoms, 1.0); c->epsilon.assign(natoms, 0.0);
        const char* pf = getenv("B200MD_PAD_FRACTION");
        if (pf) c->padFrac = atof(pf);
        const char* ug = getenv("B200MD_USE_GRAPH");
        if (ug) c->useGraph = atoi(ug) != 0;
        const char* gs = getenv("B200MD_GRAPH_STEPS");
        if (gs) c->graphSteps = std::max(1, atoi(gs));
        *out = c;
        return 0;
    } catch (std::exception& e) { g_create_error = e.what(); return -1; }
}

extern "C" void b200md_destroy(b200md_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    if (ctx->stepGraph) cudaGraphExecDestroy(ctx->stepGraph);
    if (ctx->multiGraph) cudaGraphExecDestroy(ctx->multiGraph);
    for (int q = 0; q < B200MD_MAX_RANKS; q++) if (ctx->peerMapped[q]) cudaIpcCloseMemHandle(ctx->peerMapped[q]);
    if (ctx->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(ctx->comm);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->streamPme) cudaStreamDestroy(ctx->streamPme);
    if (ctx->streamBonded) cudaStreamDestroy(ctx->streamBonded);
    if (ctx->evFork) cudaEventDestroy(ctx->evFork);
    if (ctx->evJoin) cudaEventDestroy(ctx->evJoin);
    if (ctx->evJoinBonded) cudaEventDestroy(ctx->evJoinBonded);
    if (ctx->evForkGrid) cudaEventDestroy(ctx->evForkGrid);
    char* window = ctx->window;
    delete ctx;
    if (window) cudaFree(window);
}

extern "C" int b200md_set_masses(b200md_ctx* ctx, const double* mass) {
    API_BEGIN(ctx)
    require(!ctx->finalized, "set_masses after finalize");
    ctx->mass.assign(mass, mass + ctx->natoms);
    API_END(ctx)
}

extern "C" int b200md_set_nonbonded(b200md_ctx* ctx, const b200md_nonbonded_desc* d, const double* q, const double* sig, const double* eps) {
    API_BEGIN(ctx)
    require(!ctx->finalized, "set_nonbonded after finalize");
    require(d->method != B200MD_NB_EWALD && d->method != B200MD_NB_LJPME, "nonbonded method not supported by the B200 platform (only NoCutoff, CutoffNonPeriodic, CutoffPeriodic, PME)");
    ctx->nbdesc = *d;
    ctx->haveNb = true;
    ctx->charge.assign(q, q + ctx->natoms);
    ctx->sigma.assign(sig, sig + ctx->natoms);
    ctx->epsilon.assign(eps, eps + ctx->natoms);
    ctx->dispersionCoefficient = d->dispersion_coefficient;
    API_END(ctx)
}

// The topology: every set_* call below refuses a call after finalize and a negative count.  The bonded ones also refuse an
// atom index outside [0, natoms) before they replace their term class's table, so no kernel and no host loop ever indexes
// with an unchecked atom (constraints are checked by classify_units).
static void check_set(const b200md_ctx* c, const char* call, int n) {
    if (c->finalized) throw std::runtime_error(std::string(call) + " after finalize");
    if (n < 0) throw std::runtime_error(std::string(call) + ": negative count");
}
extern "C" int b200md_set_exceptions(b200md_ctx* ctx, int n, const int* p1, const int* p2, const double* qq, const double* sig, const double* eps) {
    API_BEGIN(ctx)
    check_set(ctx, "set_exceptions", n);
    std::vector<int2> a(n); std::vector<double3> p(n);
    for (int i = 0; i < n; i++) { a[i] = make_int2(p1[i], p2[i]); p[i] = make_double3(qq[i], sig[i], eps[i]); }
    check_atoms(ctx->natoms, a, "exception");
    ctx->exc.atoms.swap(a); ctx->exc.params.swap(p);
    API_END(ctx)
}
extern "C" int b200md_set_bonds(b200md_ctx* ctx, int n, const int* p1, const int* p2, const double* len, const double* k) {
    API_BEGIN(ctx)
    check_set(ctx, "set_bonds", n);
    std::vector<int2> a(n); std::vector<double2> p(n);
    for (int i = 0; i < n; i++) { a[i] = make_int2(p1[i], p2[i]); p[i] = make_double2(len[i], k[i]); }
    ctx->bonds.set(ctx->natoms, "bond", n, a, p);
    API_END(ctx)
}
extern "C" int b200md_set_angles(b200md_ctx* ctx, int n, const int* p1, const int* p2, const int* p3, const double* t0, const double* k) {
    API_BEGIN(ctx)
    check_set(ctx, "set_angles", n);
    std::vector<int4> a(n); std::vector<double2> p(n);
    for (int i = 0; i < n; i++) { a[i] = make_int4(p1[i], p2[i], p3[i], 0); p[i] = make_double2(t0[i], k[i]); }
    ctx->angles.set(ctx->natoms, "angle", n, a, p);
    API_END(ctx)
}
extern "C" int b200md_set_torsions(b200md_ctx* ctx, int n, const int* p1, const int* p2, const int* p3, const int* p4, const int* per, const double* ph, const double* k) {
    API_BEGIN(ctx)
    check_set(ctx, "set_torsions", n);
    std::vector<int4> a(n); std::vector<double4> p(n);
    for (int i = 0; i < n; i++) { a[i] = make_int4(p1[i], p2[i], p3[i], p4[i]); p[i] = make_double4(k[i], ph[i], (double) per[i], 0); }
    ctx->torsions.set(ctx->natoms, "periodic torsion", n, a, p);
    API_END(ctx)
}
extern "C" int b200md_set_rb_torsions(b200md_ctx* ctx, int n, const int* p1, const int* p2, const int* p3, const int* p4, const double* c) {
    API_BEGIN(ctx)
    check_set(ctx, "set_rb_torsions", n);
    std::vector<int4> a(n); std::vector<double> p(c, c + 6*(size_t) n);
    for (int i = 0; i < n; i++) a[i] = make_int4(p1[i], p2[i], p3[i], p4[i]);
    ctx->rb.set(ctx->natoms, "RB torsion", n, a, p);
    API_END(ctx)
}
extern "C" int b200md_set_cmap(b200md_ctx* ctx, int nmaps, const int* size, const double* coeff, int n, const int* map, const int* atoms) {
    API_BEGIN(ctx)
    check_set(ctx, "set_cmap", std::min(nmaps, n));
    std::vector<int2> maps(nmaps); size_t patches = 0;      // per map (first patch, size); size^2 patches of 16 coefficients
    for (int m = 0; m < nmaps; m++) {
        require(size[m] > 0, "CMAP: the size of a map must be positive");
        maps[m] = make_int2((int) patches, size[m]); patches += (size_t) size[m]*size[m];
    }
    for (int i = 0; i < n; i++) require(map[i] >= 0 && map[i] < nmaps, "CMAP torsion: map index out of range");
    std::vector<int4> a(2*(size_t) n); std::vector<double> p(coeff, coeff + 16*patches);
    for (size_t d = 0; d < a.size(); d++) a[d] = make_int4(atoms[4*d], atoms[4*d+1], atoms[4*d+2], atoms[4*d+3]);
    ctx->cmap.set(ctx->natoms, "CMAP torsion", n, a, p);
    ctx->cmap.map.assign(map, map + n); ctx->cmap.maps.swap(maps);
    API_END(ctx)
}
// A custom-torsion program set (b200md_set_custom_torsions): prog_start well formed and every program passing
// custom_check_program (nglobals < 0: GLOBAL operands are checked at finalize).  Returns the instructions as (opcode, operand).
static std::vector<int2> check_programs(int nprog, const int* prog_start, const int* op, const int* arg, int stride, int nglobals) {
    require(nprog >= 0, "set_custom_torsions: negative number of programs");
    require(stride >= 0 && stride <= B200MD_CUSTOM_MAX_PARAMS, "set_custom_torsions: more than 16 parameters per torsion");
    require(nprog == 0 || prog_start[0] == 0, "set_custom_torsions: prog_start[0] must be 0");
    for (int q = 0; q < 2*nprog; q++) require(prog_start[q+1] >= prog_start[q], "set_custom_torsions: prog_start must not decrease");
    const int total = nprog ? prog_start[2*nprog] : 0;
    std::vector<int2> code(total);
    for (int k = 0; k < total; k++) code[k] = make_int2(op[k], arg[k]);
    for (int q = 0; q < 2*nprog; q++) {
        const char* why = custom_check_program(code.data(), prog_start[q], prog_start[q+1], stride, nglobals);
        if (why) throw std::runtime_error(std::string(why) + " (program " + std::to_string(q) + ")");
    }
    return code;
}
extern "C" int b200md_set_custom_torsions(b200md_ctx* ctx, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                          int stride, int n, const int* prog, const int* atoms, const double* params) {
    API_BEGIN(ctx)
    check_set(ctx, "set_custom_torsions", n);
    require(ctx->world == 1, "custom torsions are not supported in multi-GPU runs");
    std::vector<int2> code = check_programs(nprog, prog_start, op, arg, stride, -1);
    for (int i = 0; i < n; i++) require(prog[i] >= 0 && prog[i] < nprog, "custom torsion: program index out of range");
    std::vector<int4> a(n); std::vector<double> p(params, params + (size_t) n*stride);
    for (int i = 0; i < n; i++) a[i] = make_int4(atoms[4*i], atoms[4*i+1], atoms[4*i+2], atoms[4*i+3]);
    CustomTorsionTable& t = ctx->custom;
    t.set(ctx->natoms, "custom torsion", n, a, p);
    t.stride = stride; t.nprog = nprog; t.code.swap(code);
    t.imm.assign(imm, imm + t.code.size()); t.progStart.assign(prog_start, prog_start + (nprog ? 2*nprog + 1 : 0)); t.prog.assign(prog, prog + n);
    API_END(ctx)
}
extern "C" int b200md_set_custom_globals(b200md_ctx* ctx, int n, const double* values) {
    API_BEGIN(ctx)
    require(n >= 0, "set_custom_globals: negative count");
    CustomTorsionTable& t = ctx->custom;
    if (!ctx->finalized) { t.globals.assign(values, values + n); return 0; }
    require(n == (int) t.globals.size(), "set_custom_globals: the number of global parameters cannot change after finalize");
    t.globals.assign(values, values + n);
    // stream ordered, into the buffer the step graphs read: no graph is captured or instantiated again
    if (n) CUDA_CHECK(cudaMemcpyAsync(t.globalsDev.p, t.globals.data(), sizeof(double)*n, cudaMemcpyHostToDevice, ctx->stream));
    API_END(ctx)
}
extern "C" int b200md_custom_program_probe(int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                           int stride, int nglobals, int which, double theta, const double* params,
                                           const double* globals, double* out, char* msg, int msglen) {
    try {
        require(nglobals >= 0, "custom_program_probe: negative number of globals");
        const std::vector<int2> code = check_programs(nprog, prog_start, op, arg, stride, nglobals);
        require(which >= 0 && which < 2*nprog, "custom_program_probe: program index out of range");
        *out = custom_run(code.data(), imm, prog_start[which], prog_start[which+1], theta, params, globals);
        return 0;
    } catch (std::exception& e) {
        if (msg && msglen > 0) { strncpy(msg, e.what(), msglen - 1); msg[msglen - 1] = 0; }
        return -1;
    }
}
extern "C" int b200md_set_bonded_groups(b200md_ctx* ctx, int kind, int n, const int* group) {
    API_BEGIN(ctx)
    check_set(ctx, "set_bonded_groups", n);
    require(kind >= B200MD_BONDED_BONDS && kind <= B200MD_BONDED_CUSTOM_TORSIONS,
            "set_bonded_groups: kind must be 0 (bonds), 1 (angles), 2 (torsions), 3 (RB torsions), 4 (CMAP) or 5 (custom torsions)");
    std::vector<unsigned char>& g = kind == B200MD_BONDED_BONDS ? ctx->bonds.group : kind == B200MD_BONDED_ANGLES ? ctx->angles.group :
                                    kind == B200MD_BONDED_TORSIONS ? ctx->torsions.group : kind == B200MD_BONDED_RB_TORSIONS ? ctx->rb.group :
                                    kind == B200MD_BONDED_CMAP ? ctx->cmap.group : ctx->custom.group;
    g.resize(n);
    for (int i = 0; i < n; i++) { require(group[i] >= 0 && (group[i] & ~0x80) < 32, "force group out of range"); g[i] = (unsigned char) group[i]; }
    API_END(ctx)
}
extern "C" int b200md_set_constraints(b200md_ctx* ctx, int n, const int* p1, const int* p2, const double* d) {
    API_BEGIN(ctx)
    check_set(ctx, "set_constraints", n);
    ctx->conI.assign(p1, p1+n); ctx->conJ.assign(p2, p2+n); ctx->conD.assign(d, d+n);
    API_END(ctx)
}
extern "C" int b200md_set_cm_remover(b200md_ctx* ctx, int freq) {
    if (!ctx) return -1;
    ctx->cmFreq = freq;
    return 0;
}

extern "C" int b200md_set_precision(b200md_ctx* ctx, int precision) {
    API_BEGIN(ctx)
    require(!ctx->finalized, "set_precision after finalize");
    require(precision == B200MD_PRECISION_SINGLE || precision == B200MD_PRECISION_MIXED,
            "set_precision: unknown precision (B200MD_PRECISION_SINGLE or B200MD_PRECISION_MIXED)");
    require(precision == B200MD_PRECISION_SINGLE || ctx->world == 1, "mixed precision is not supported in multi-GPU runs");
    require(precision == B200MD_PRECISION_SINGLE || !ctx->pmeOnly, "mixed precision is not supported by the stand-alone PME provider");
    ctx->precision = precision;
    API_END(ctx)
}
extern "C" int b200md_get_precision(b200md_ctx* ctx) { return ctx ? ctx->precision : -1; }

extern "C" int b200md_remove_cm_motion(b200md_ctx* ctx) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    require(ctx->finalized, "remove_cm_motion before finalize");
    sync_velocities(ctx);
    launch_remove_cm(ctx->nb, ctx->cmScratch.p, ctx->stream);
    ctx->kernelLaunches += 2;
    API_END(ctx)
}

// ---------------------------------------------------------------- space-filling order of the binning cells
// Blocked serpentine: 2x2x2 super-cells visited in a 3-D boustrophedon (every step of the path moves to a face-adjacent
// super-cell), cells inside a super-cell in a fixed order.  Unlike a Hilbert / Morton curve restricted to a
// non-power-of-two grid, the path never leaves and re-enters the grid, so 32 consecutive sorted atoms (~ one super-cell
// at ~4 atoms per cell) always form a compact ~2x2x2-cell cube.  (Round 1 used a Hilbert curve on the padded 2^k grid:
// the blocks that straddled its re-entry points had bounding boxes of nanometres, which switched the tile kernel's
// single-image mode off and wasted tile slots.)
static void cell_order(const int nc[3], std::vector<int>& rank) {
    const int sx = (nc[0] + 1)/2, sy = (nc[1] + 1)/2, sz = (nc[2] + 1)/2;
    rank.assign((size_t) nc[0]*nc[1]*nc[2], 0);
    int r = 0;
    for (int ix = 0; ix < sx; ix++)
        for (int jy = 0; jy < sy; jy++) {
            const int iy = (ix & 1) ? sy-1-jy : jy;
            for (int kz = 0; kz < sz; kz++) {
                const int iz = ((ix*sy + jy) & 1) ? sz-1-kz : kz;
                for (int a = 0; a < 2; a++) for (int b = 0; b < 2; b++) for (int c = 0; c < 2; c++) {
                    const int x = 2*ix + a, y = 2*iy + b, z = 2*iz + c;
                    if (x < nc[0] && y < nc[1] && z < nc[2]) rank[((size_t) x*nc[1] + y)*nc[2] + z] = r++;
                }
            }
        }
}

static void setup_cells(b200md_ctx* c) {
    int nc[3] = {1, 1, 1};
    if (c->nb.box.periodic) {
        const double vol = c->boxA[0]*c->boxB[1]*c->boxC[2];
        const double density = c->natoms/vol;
        double edge = std::cbrt(4.0/density);
        const double L[3] = {c->boxA[0], c->boxB[1], c->boxC[2]};
        for (int d = 0; d < 3; d++) nc[d] = std::max(1, std::min(128, (int) std::floor(L[d]/edge)));
    }
    const int ncells = nc[0]*nc[1]*nc[2];
    if (ncells != c->nb.ncells || nc[0] != c->nb.ncell[0] || nc[1] != c->nb.ncell[1] || nc[2] != c->nb.ncell[2]) {
        std::vector<int> rank;
        cell_order(nc, rank);
        c->cellRank.upload(rank);
        c->cellCount.alloc(ncells + 1); c->cellCount.zero();     // every list build leaves them zeroed again (k_list_prep)
        c->cellFill.alloc(ncells); c->cellFill.zero();
        c->nb.ncells = ncells;
        for (int d = 0; d < 3; d++) c->nb.ncell[d] = nc[d];
        c->nb.cellRank = c->cellRank.p; c->nb.cellCount = c->cellCount.p; c->nb.cellFill = c->cellFill.p;
    }
}

// The step graphs hold kernel parameters by value (box, tile-pool pointers, cell grid, integrator constants): whatever changes
// one of them marks both graphs stale.  b200md_step captures them again and updates the executable graphs in place
// (capture_steps), so a box change every few steps -- a barostat -- does not instantiate graphs.
static void invalidate_graph(b200md_ctx* c) { c->graphValid = false; c->multiValid = false; }

static void set_counter(b200md_ctx* c, int index, int value) {
    CUDA_CHECK(cudaMemcpyAsync(&c->counters.p[index], &value, sizeof(int), cudaMemcpyHostToDevice, c->stream));
}
// The state was changed from outside: the next evaluation rebuilds the list, synchronously and before any step graph
// (prepare_list), which then trusts it.
static void request_rebuild(b200md_ctx* c) { set_counter(c, CT_REBUILD, 1); c->listDirty = true; }

static void apply_box(b200md_ctx* c) {
    BoxDev& b = c->nb.box;
    const int m = c->nbdesc.method;
    b.periodic = (m == B200MD_NB_CUTOFF_PERIODIC || m == B200MD_NB_PME) ? 1 : 0;
    if (c->haveBox) {
        b.ax = (float) c->boxA[0]; b.bx = (float) c->boxB[0]; b.by = (float) c->boxB[1];
        b.cx = (float) c->boxC[0]; b.cy = (float) c->boxC[1]; b.cz = (float) c->boxC[2];
        b.invAx = (float) (1.0/c->boxA[0]); b.invBy = (float) (1.0/c->boxB[1]); b.invCz = (float) (1.0/c->boxC[2]);
        b.dax = c->boxA[0]; b.dby = c->boxB[1]; b.dcz = c->boxC[2];
        b.triclinic = (c->boxB[0] != 0 || c->boxC[0] != 0 || c->boxC[1] != 0) ? 1 : 0;
        const double det = c->boxA[0]*c->boxB[1]*c->boxC[2];
        const double s = 1.0/det;
        double* R = b.recip;       // invert_box_vectors, ReferencePME.cpp:196-204
        R[0] = c->boxB[1]*c->boxC[2]*s; R[1] = 0; R[2] = 0;
        R[3] = -c->boxB[0]*c->boxC[2]*s; R[4] = c->boxA[0]*c->boxC[2]*s; R[5] = 0;
        R[6] = (c->boxB[0]*c->boxC[1] - c->boxB[1]*c->boxC[0])*s; R[7] = -c->boxA[0]*c->boxC[1]*s; R[8] = c->boxA[0]*c->boxB[1]*s;
        b.volume = det;
    }
    else {
        require(!b.periodic, "periodic nonbonded method needs box vectors (b200md_set_box)");
        b.ax = b.by = b.cz = 1.f; b.bx = b.cx = b.cy = 0.f; b.invAx = b.invBy = b.invCz = 1.f; b.triclinic = 0; b.dax = b.dby = b.dcz = 1;
        for (int i = 0; i < 9; i++) b.recip[i] = 0; b.volume = 1;
    }
    if (b.periodic) {
        const double rc = c->nbdesc.cutoff;
        require(c->boxA[0] >= 1.999999*rc && c->boxB[1] >= 1.999999*rc && c->boxC[2] >= 1.999999*rc,
                "The periodic box size has decreased to less than twice the nonbonded cutoff.");   // ReferenceKernels.cpp:983-985
    }
    if (c->finalized) {
        setup_cells(c);
        if (m == B200MD_NB_PME) { launch_pme_eterm(c->nb, c->pme, c->stream); c->kernelLaunches++; }
        request_rebuild(c);
        CUDA_CHECK(cudaStreamSynchronize(c->stream));
        invalidate_graph(c);
    }
}

extern "C" int b200md_set_box(b200md_ctx* ctx, const double a[3], const double b[3], const double c[3]) {
    API_BEGIN(ctx)
    for (int i = 0; i < 3; i++) { ctx->boxA[i] = a[i]; ctx->boxB[i] = b[i]; ctx->boxC[i] = c[i]; }
    ctx->haveBox = true;
    if (ctx->finalized) apply_box(ctx);
    API_END(ctx)
}
extern "C" int b200md_get_box(b200md_ctx* ctx, double a[3], double b[3], double c[3]) {
    if (!ctx) return -1;
    for (int i = 0; i < 3; i++) { a[i] = ctx->boxA[i]; b[i] = ctx->boxB[i]; c[i] = ctx->boxC[i]; }
    return 0;
}

// ---------------------------------------------------------------- the per-atom dynamic state
enum { ST_POS = 1, ST_VEL = 2, ST_CELL = 4, ST_ALL = 7 };
// The context's state arrays for its precision, in checkpoint order: posq | posqCorr (mixed) | velm (single) or velmD
// (mixed) | cellOffset.  `what` selects the positions, the velocities and cellOffset.
static std::vector<DevSpan> state_spans(const b200md_ctx* c, int what = ST_ALL) {
    const size_t NP = c->npad;
    std::vector<DevSpan> s;
    if (what & ST_POS) {
        s.push_back({c->posq.p, sizeof(float4)*NP});
        if (c->mixed()) s.push_back({c->posqCorr.p, sizeof(float4)*NP});
    }
    if (what & ST_VEL) s.push_back(c->mixed() ? DevSpan{c->velmD.p, sizeof(double4)*NP} : DevSpan{c->velm.p, sizeof(float4)*NP});
    if (what & ST_CELL) s.push_back({c->cellOffset.p, sizeof(int)*3*NP});
    return s;
}

// Velocities v (nullptr: zero) with 1/mass in w (0 for a massless atom), into velm (V = float4) or velmD (V = double4).
template <class V> static void upload_velocities(b200md_ctx* c, V* dst, const double* v) {
    typedef decltype(V::x) E;
    const double none[3] = {0, 0, 0};
    std::vector<V> h(c->npad, V{});
    for (int i = 0; i < c->natoms; i++) {
        const double* u = v ? v + 3*i : none;
        h[i] = V{(E) u[0], (E) u[1], (E) u[2], c->mass[i] > 0 ? (E) (1.0/c->mass[i]) : (E) 0};
    }
    CUDA_CHECK(cudaMemcpyAsync(dst, h.data(), sizeof(V)*c->npad, cudaMemcpyHostToDevice, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
}

// ---------------------------------------------------------------- Monte Carlo barostat
// ApplyMonteCarloBarostatKernel (kernels.h:1425-1459).  The host half (MonteCarloBarostatImpl: random volume change, the two
// energy evaluations, acceptance, adaptive step) stays the reference's own; these three calls are the platform's part.
static void require_single_rank(const b200md_ctx* c, const char* what) {
    if (c->world > 1) throw std::runtime_error(std::string(what) + ": the Monte Carlo barostat is not supported in multi-GPU runs");
}

extern "C" int b200md_set_barostat_molecules(b200md_ctx* ctx, int nmol, const int* start, const int* atoms) {
    API_BEGIN(ctx)
    require_single_rank(ctx, "set_barostat_molecules");
    require(nmol >= 0 && start != nullptr && start[0] == 0 && start[nmol] <= ctx->natoms && (start[nmol] == 0 || atoms != nullptr),
            "set_barostat_molecules: malformed molecule list");
    for (int m = 0; m < nmol; m++) require(start[m+1] > start[m], "set_barostat_molecules: empty molecule");
    for (int t = 0; t < start[nmol]; t++) require(atoms[t] >= 0 && atoms[t] < ctx->natoms, "set_barostat_molecules: atom index out of range");
    ctx->baroStart.upload(std::vector<int>(start, start + nmol + 1));
    ctx->baroAtoms.upload(std::vector<int>(atoms, atoms + start[nmol]));
    ctx->baroNmol = nmol;
    API_END(ctx)
}

extern "C" int b200md_scale_coordinates(b200md_ctx* ctx, double sx, double sy, double sz) {
    API_BEGIN(ctx)
    b200md_ctx* c = ctx;
    require_single_rank(c, "scale_coordinates");
    require(c->finalized && c->haveBox, "scale_coordinates before finalize / set_box");
    require(c->baroStart.n > 0, "scale_coordinates before set_barostat_molecules");
    // the velocities are not saved: the move does not touch them
    c->baroSave.parts = state_spans(c, ST_POS | ST_CELL);
    c->baroSave.parts.push_back({c->force.p, sizeof(long long)*3*c->npad});
    c->baroSave.save(c->stream);
    ScaleDev sc{};
    sc.nmol = c->baroNmol; sc.molStart = c->baroStart.p; sc.molAtoms = c->baroAtoms.p;
    for (int k = 0; k < 3; k++) { sc.a[k] = c->boxA[k]; sc.b[k] = c->boxB[k]; sc.c[k] = c->boxC[k]; }
    sc.s[0] = sx; sc.s[1] = sy; sc.s[2] = sz;
    launch_scale_molecules(c->nb, sc, c->stream);
    c->kernelLaunches++;
    CUDA_CHECK(cudaGetLastError());
    request_rebuild(c);
    c->stepStateValid = false;
    API_END(ctx)
}

extern "C" int b200md_restore_coordinates(b200md_ctx* ctx) {
    API_BEGIN(ctx)
    b200md_ctx* c = ctx;
    require_single_rank(c, "restore_coordinates");
    require(!c->baroSave.parts.empty(), "restore_coordinates without a preceding scale_coordinates");
    c->baroSave.restore(c->stream);
    request_rebuild(c);
    c->stepStateValid = false;            // the force buffer holds forces again, not the zeros the fused step expects
    API_END(ctx)
}

// per-atom and per-exception parameters -> device (computeParameters, ReferenceKernels.cpp:1077-1121)
static void upload_params(b200md_ctx* c) {
    const int N = c->natoms;
    const double sk = std::sqrt(B200MD_ONE_4PI_EPS0);
    std::vector<float2> se(c->npad, make_float2(0.f, 0.f));
    for (int i = 0; i < N; i++) se[i] = make_float2((float) (0.5*c->sigma[i]), (float) (2.0*std::sqrt(c->epsilon[i])));
    c->sigeps.upload(se);
    {
        std::vector<double> qd(c->npad, 0.0); std::vector<double2> sd(c->npad, make_double2(0.0, 0.0));
        for (int i = 0; i < N; i++) { qd[i] = c->charge[i]*sk; sd[i] = make_double2(0.5*c->sigma[i], 2.0*std::sqrt(c->epsilon[i])); }
        c->chargeD.upload(qd); c->sigepsD.upload(sd);
        c->nb.chargeD = c->pmeOnly ? nullptr : c->chargeD.p; c->nb.sigepsD = c->sigepsD.p;     // stand-alone PME: the charges arrive with every call (posq.w)
    }
    // charges live in posq.w; keep positions
    std::vector<float4> p(c->npad);
    CUDA_CHECK(cudaMemcpy(p.data(), c->posq.p, sizeof(float4)*c->npad, cudaMemcpyDeviceToHost));
    for (int i = 0; i < N; i++) p[i].w = (float) (c->charge[i]*sk);
    CUDA_CHECK(cudaMemcpy(c->posq.p, p.data(), sizeof(float4)*c->npad, cudaMemcpyHostToDevice));
    const int ne = (int) c->exc.atoms.size();
    std::vector<double4> ep(ne);
    for (int e = 0; e < ne; e++) {
        const int2 a = c->exc.atoms[e]; const double3 p = c->exc.params[e];
        ep[e] = make_double4(B200MD_ONE_4PI_EPS0*p.x, p.y, 4.0*p.z, B200MD_ONE_4PI_EPS0*c->charge[a.x]*c->charge[a.y]);
    }
    c->exc.atomsDev.upload(c->exc.atoms); c->exc.paramsDev.upload(ep);
    c->bd.nexc = ne; c->bd.excAtoms = c->exc.atomsDev.p; c->bd.excParams = c->exc.paramsDev.p;
    double self = 0;
    if (c->nbdesc.method == B200MD_NB_PME)
        for (int i = 0; i < N; i++) self -= B200MD_ONE_4PI_EPS0*c->charge[i]*c->charge[i]*c->nbdesc.ewald_alpha/std::sqrt(M_PI);
    c->selfEnergy = self;
}

// Integration units: SETTLE waters, X-H_n SHAKE clusters, free atoms.  Pure host function so that the plugin can run it
// as a dry run from Platform::contextCreated (b200md_check_constraints) before anything is allocated.
static bool classify_units(int N, const double* mass, const std::vector<int>& conI, const std::vector<int>& conJ, const std::vector<double>& conD,
                           std::vector<int4>& ua2, std::vector<int>& ut2, std::vector<float4>& up2, std::string& err, std::vector<int>* ccmaCons = nullptr,
                           std::vector<double4>* upD2 = nullptr) {
    const int nc = (int) conI.size();
    std::vector<std::vector<std::pair<int, double> > > adj(N);
    for (int k = 0; k < nc; k++) {
        if (conI[k] < 0 || conI[k] >= N || conJ[k] < 0 || conJ[k] >= N || conI[k] == conJ[k]) { err = "constraint with an illegal particle index"; return false; }
        if (mass[conI[k]] == 0 && mass[conJ[k]] == 0) continue;           // constraints between immovable particles are ignored (ReferenceConstraints.cpp:60)
        if (mass[conI[k]] == 0 || mass[conJ[k]] == 0) { err = "A constraint cannot involve a massless particle"; return false; }      // ContextImpl.cpp:86-87
        adj[conI[k]].push_back(std::make_pair(conJ[k], conD[k]));
        adj[conJ[k]].push_back(std::make_pair(conI[k], conD[k]));
    }
    std::vector<int> assigned(N, 0);
    std::vector<int4> ua; std::vector<int> ut; std::vector<float4> up; std::vector<double4> upD;     // upD: the distances in double
    std::vector<std::pair<int, int> > order;      // (first atom, unit index) for sorting
    auto dist = [&](int a, int b) -> double { for (auto& pr : adj[a]) if (pr.first == b) return pr.second; return -1.0; };
    // SETTLE: closed triangles with two equal sides (compared as float, ReferenceConstraints.cpp:73-77,111-137)
    for (int a = 0; a < N; a++) {
        if (assigned[a] || adj[a].size() != 2) continue;
        int b = adj[a][0].first, d = adj[a][1].first;
        if (adj[b].size() != 2 || adj[d].size() != 2 || assigned[b] || assigned[d]) continue;
        if (dist(b, d) < 0) continue;
        const float dab = (float) dist(a, b), dad = (float) dist(a, d), dbd = (float) dist(b, d);
        int apex, o1, o2; float d1, d2; double d1D, d2D;
        if (dab == dad) { apex = a; o1 = b; o2 = d; d1 = dab; d2 = dbd; d1D = dist(a, b); d2D = dist(b, d); }
        else if (dab == dbd) { apex = b; o1 = a; o2 = d; d1 = dab; d2 = dad; d1D = dist(a, b); d2D = dist(a, d); }
        else if (dad == dbd) { apex = d; o1 = a; o2 = b; d1 = dad; d2 = dab; d1D = dist(a, d); d2D = dist(a, b); }
        else continue;
        if (mass[apex] == 0 || mass[o1] == 0 || mass[o2] == 0) continue;
        assigned[a] = assigned[b] = assigned[d] = 1;
        order.push_back(std::make_pair(std::min(a, std::min(b, d)), (int) ua.size()));
        ua.push_back(make_int4(apex, o1, o2, -1)); ut.push_back(1); up.push_back(make_float4(d1, d2, 0.f, 0.f)); upD.push_back(make_double4(d1D, d2D, 0, 0));
    }
    // SHAKE clusters: a centre whose partners are each constrained only to it (IntegrationUtilities.cpp:204-277)
    for (int a = 0; a < N; a++) {
        if (assigned[a] || adj[a].empty()) continue;
        bool centre = adj[a].size() <= 3;
        for (auto& pr : adj[a]) if (adj[pr.first].size() != 1 || assigned[pr.first]) centre = false;
        if (adj[a].size() == 1 && adj[adj[a][0].first].size() == 1) {
            // isolated pair: the heavier atom is the centre, ties -> lower index
            int b = adj[a][0].first;
            if (mass[b] > mass[a] || (mass[b] == mass[a] && b < a)) centre = false;
        }
        if (!centre) continue;
        int at[4] = {a, -1, -1, -1}; float dd[3] = {0, 0, 0}; double ddD[3] = {0, 0, 0};
        for (size_t k = 0; k < adj[a].size(); k++) { at[k+1] = adj[a][k].first; dd[k] = (float) adj[a][k].second; ddD[k] = adj[a][k].second; assigned[adj[a][k].first] = 1; }
        assigned[a] = 1;
        order.push_back(std::make_pair(a, (int) ua.size()));
        ua.push_back(make_int4(at[0], at[1], at[2], at[3])); ut.push_back(2); up.push_back(make_float4(dd[0], dd[1], dd[2], 0.f)); upD.push_back(make_double4(ddD[0], ddD[1], ddD[2], 0));
    }
    // everything else is a general constraint network: CCMA (ReferenceConstraints.cpp:148-184).  Its atoms get no
    // integration unit: k_ccma_step (constraints.cu) takes them through the step, one CTA per connected component.
    std::vector<char> isCcma(N, 0);
    for (int a = 0; a < N; a++) if (!assigned[a] && !adj[a].empty()) {
        isCcma[a] = 1;
    }
    if (ccmaCons) {
        ccmaCons->clear();
        for (int k = 0; k < nc; k++) if ((isCcma[conI[k]] || isCcma[conJ[k]]) && mass[conI[k]] != 0) ccmaCons->push_back(k);
    }
    for (int a = 0; a < N; a++) {
        if (isCcma[a]) continue;
        if (!assigned[a]) {
            order.push_back(std::make_pair(a, (int) ua.size()));
            ua.push_back(make_int4(a, -1, -1, -1)); ut.push_back(0); up.push_back(make_float4(0, 0, 0, 0)); upD.push_back(make_double4(0, 0, 0, 0));
        }
    }
    std::sort(order.begin(), order.end());
    ua2.resize(ua.size()); ut2.resize(ua.size()); up2.resize(ua.size());
    for (size_t k = 0; k < order.size(); k++) { ua2[k] = ua[order[k].second]; ut2[k] = ut[order[k].second]; up2[k] = up[order[k].second]; }
    if (upD2) { upD2->resize(ua.size()); for (size_t k = 0; k < order.size(); k++) (*upD2)[k] = upD[order[k].second]; }
    return true;
}

static void build_units(b200md_ctx* c) {
    std::vector<int4> ua2; std::vector<int> ut2; std::vector<float4> up2; std::vector<double4> upD2;
    std::string err;
    if (!classify_units(c->natoms, c->mass.data(), c->conI, c->conJ, c->conD, ua2, ut2, up2, err, &c->ccmaCons, &upD2)) throw std::runtime_error("B200 platform: " + err);
    c->unitAtoms.upload(ua2); c->unitType.upload(ut2); c->unitParams.upload(up2);
    if (c->mixed()) c->unitParamsD.upload(upD2);
    c->units.unitParamsD = c->mixed() ? c->unitParamsD.p : nullptr;
    c->hUnitAtoms = ua2;
    c->units.nunits = (int) ua2.size();
    c->units.unitAtoms = c->unitAtoms.p; c->units.unitType = c->unitType.p; c->units.unitParams = c->unitParams.p;
}

// ---------------------------------------------------------------- CCMA setup (host)
// Coupling matrix exactly as ReferenceCCMAAlgorithm's constructor builds it (ReferenceCCMAAlgorithm.cpp:73-135: constraints
// j, k that share an atom couple with scale * cos(angle), the angle from a third constraint that closes the triangle or
// else from a HarmonicAngleForce term); its inverse is then APPROXIMATED column by column from the constraints within three
// bonds of the column's constraint (a dense solve of ~50-100 unknowns) instead of the reference's global sparse QR
// (:137-190, QUERN): the inverse decays by ~3x per bond, entries below the reference's cut-off 0.02 (ReferenceConstraints.cpp:183)
// are dropped either way, and CCMA only needs an approximate inverse -- it iterates to the tolerance.
// host-side result of the CCMA setup; pure function of the System (no device), so that it can be probed on a CPU
// (b200md_ccma_setup_probe, tests/test_ccma_cpu.py)
struct CcmaInput {
    int natoms;
    const std::vector<double>& mass;
    const std::vector<int>& ccmaCons; const std::vector<int>& conI; const std::vector<int>& conJ; const std::vector<double>& conD;
    const std::vector<int4>& angAtoms; const std::vector<double2>& angParams;     // the layout of b200md_ctx::angles
};
struct CcmaHost {
    int ncomp = 0;
    std::vector<int> order, compCon, compAtom, atoms, aStart, aCon, rowStart, col;
    std::vector<int2> conAtoms; std::vector<float> dist, redMass, val;
    std::vector<double> distD, redMassD;     // the same in double (mixed precision)
};
static void ccma_host_setup(const CcmaInput* c, CcmaHost& H) {
    const int nc = (int) c->ccmaCons.size();
    const int N = c->natoms;
    // ---- components ----
    std::vector<int> parent(N);
    for (int i = 0; i < N; i++) parent[i] = i;
    auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
    for (int k : c->ccmaCons) { int a = find(c->conI[k]), b = find(c->conJ[k]); if (a != b) parent[std::max(a, b)] = std::min(a, b); }
    std::vector<int> order(nc);
    for (int k = 0; k < nc; k++) order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return find(c->conI[c->ccmaCons[a]]) < find(c->conI[c->ccmaCons[b]]); });
    std::vector<int2> conAtoms(nc); std::vector<float> dist(nc), redMass(nc); std::vector<double> distD(nc), redMassD(nc);
    std::vector<int> compCon(1, 0), compOfCon(nc);
    for (int k = 0; k < nc; k++) {
        const int src = c->ccmaCons[order[k]];
        conAtoms[k] = make_int2(c->conI[src], c->conJ[src]);
        distD[k] = c->conD[src]; dist[k] = (float) distD[k];
        redMassD[k] = 0.5/(1.0/c->mass[conAtoms[k].x] + 1.0/c->mass[conAtoms[k].y]);
        redMass[k] = (float) redMassD[k];
        if (k > 0 && find(conAtoms[k].x) != find(conAtoms[k-1].x)) compCon.push_back(k);
        compOfCon[k] = (int) compCon.size() - 1;
    }
    compCon.push_back(nc);
    const int ncomp = (int) compCon.size() - 1;
    // ---- atoms per component, atom -> constraints ----
    std::vector<std::vector<int> > atomCons(N);
    for (int k = 0; k < nc; k++) { atomCons[conAtoms[k].x].push_back(k + 1); atomCons[conAtoms[k].y].push_back(-(k + 1)); }
    std::vector<int> atoms, compAtom(1, 0), aStart(1, 0), aCon;
    for (int cidx = 0; cidx < ncomp; cidx++) {
        std::set<int> as;
        for (int k = compCon[cidx]; k < compCon[cidx+1]; k++) { as.insert(conAtoms[k].x); as.insert(conAtoms[k].y); }
        for (int a : as) { atoms.push_back(a); aCon.insert(aCon.end(), atomCons[a].begin(), atomCons[a].end()); aStart.push_back((int) aCon.size()); }
        compAtom.push_back((int) atoms.size());
    }
    // ---- coupling matrix ----
    std::vector<std::vector<int> > atomAngles(N);
    for (size_t i = 0; i < c->angAtoms.size(); i++) atomAngles[c->angAtoms[i].y].push_back((int) i);
    std::vector<std::vector<std::pair<int, double> > > M(nc);
    auto consOf = [&](int a) { std::vector<int> v; for (int code : atomCons[a]) v.push_back(std::abs(code) - 1); return v; };
    for (int j = 0; j < nc; j++) {
        const int j0 = conAtoms[j].x, j1 = conAtoms[j].y;
        const double w0 = 1.0/c->mass[j0], w1 = 1.0/c->mass[j1];
        std::set<int> nbrs;
        for (int k : consOf(j0)) nbrs.insert(k);
        for (int k : consOf(j1)) nbrs.insert(k);
        for (int k : nbrs) {
            if (k == j) { M[j].push_back(std::make_pair(j, 1.0)); continue; }
            const int k0 = conAtoms[k].x, k1 = conAtoms[k].y;
            int aa, ab, ac; double scale;
            if (j0 == k0) { aa = j1; ab = j0; ac = k1; scale = w0/(w0+w1); }
            else if (j1 == k1) { aa = j0; ab = j1; ac = k0; scale = w1/(w0+w1); }
            else if (j0 == k1) { aa = j1; ab = j0; ac = k0; scale = w0/(w0+w1); }
            else if (j1 == k0) { aa = j0; ab = j1; ac = k1; scale = w1/(w0+w1); }
            else continue;
            bool found = false;
            for (int other : consOf(aa))
                if (conAtoms[other].x == ac || conAtoms[other].y == ac) {
                    const double d1 = distD[j], d2 = distD[k], d3 = distD[other];
                    M[j].push_back(std::make_pair(k, scale*(d1*d1 + d2*d2 - d3*d3)/(2.0*d1*d2)));
                    found = true;
                    break;
                }
            if (!found)
                for (int cand : atomAngles[ab])
                    if ((c->angAtoms[cand].x == aa && c->angAtoms[cand].z == ac) || (c->angAtoms[cand].z == aa && c->angAtoms[cand].x == ac)) {
                        M[j].push_back(std::make_pair(k, scale*std::cos(c->angParams[cand].x)));
                        break;
                    }
        }
    }
    // ---- approximate inverse, column by column ----
    std::vector<std::vector<std::pair<int, float> > > inv(nc);      // inv[row] = (col, value)
    std::vector<std::vector<std::pair<int, float> > > colOut(nc);   // per column: (row, value), filled in parallel
    auto solve_columns = [&](int begin, int end) {
        std::vector<int> S, localOf(nc, -1);
        std::vector<double> A, x;
        for (int i = begin; i < end; i++) {
            // constraints within 3 bonds of constraint i (breadth first over "shares an atom"), at most 160
            S.assign(1, i); localOf[i] = 0;
            size_t head = 0; int depthEnd = 1, depth = 0;
            while (head < S.size() && depth < 3 && S.size() < 160) {
                const int k = S[head++];
                for (auto& el : M[k]) if (localOf[el.first] < 0 && S.size() < 160) { localOf[el.first] = (int) S.size(); S.push_back(el.first); }
                if ((int) head == depthEnd) { depth++; depthEnd = (int) S.size(); }
            }
            const int n = (int) S.size();
            A.assign((size_t) n*n, 0.0); x.assign(n, 0.0); x[0] = 1.0;
            for (int r = 0; r < n; r++) for (auto& el : M[S[r]]) if (localOf[el.first] >= 0) A[(size_t) r*n + localOf[el.first]] = el.second;
            for (int p = 0; p < n; p++) {              // Gaussian elimination with partial pivoting
                int piv = p;
                for (int r = p+1; r < n; r++) if (std::fabs(A[(size_t) r*n + p]) > std::fabs(A[(size_t) piv*n + p])) piv = r;
                if (piv != p) { for (int q = 0; q < n; q++) std::swap(A[(size_t) p*n + q], A[(size_t) piv*n + q]); std::swap(x[p], x[piv]); }
                const double d = A[(size_t) p*n + p];
                if (d == 0.0) continue;
                for (int r = p+1; r < n; r++) {
                    const double f = A[(size_t) r*n + p]/d;
                    if (f == 0.0) continue;
                    for (int q = p; q < n; q++) A[(size_t) r*n + q] -= f*A[(size_t) p*n + q];
                    x[r] -= f*x[p];
                }
            }
            for (int p = n-1; p >= 0; p--) {
                double sacc = x[p];
                for (int q = p+1; q < n; q++) sacc -= A[(size_t) p*n + q]*x[q];
                x[p] = (A[(size_t) p*n + p] != 0.0) ? sacc/A[(size_t) p*n + p] : 0.0;
            }
            for (int r = 0; r < n; r++) {
                const int j = S[r];
                const double value = x[r]*distD[i]/distD[j];            // ReferenceCCMAAlgorithm.cpp:177
                if (std::fabs(value) > 0.02) colOut[i].push_back(std::make_pair(j, (float) value));
                localOf[j] = -1;
            }
        }
    };
    {
        const int nthreads = std::max(1, std::min(16, (int) std::thread::hardware_concurrency()));
        std::vector<std::thread> pool;
        for (int t = 0; t < nthreads; t++) pool.emplace_back(solve_columns, (int) ((long long) nc*t/nthreads), (int) ((long long) nc*(t+1)/nthreads));
        for (auto& th : pool) th.join();
    }
    for (int i = 0; i < nc; i++) for (auto& el : colOut[i]) inv[el.first].push_back(std::make_pair(i, el.second));
    std::vector<int> rowStart(1, 0), col; std::vector<float> val;
    for (int j = 0; j < nc; j++) { for (auto& el : inv[j]) { col.push_back(el.first); val.push_back(el.second); } rowStart.push_back((int) col.size()); }
    H.ncomp = ncomp;
    H.order = order; H.compCon = compCon; H.compAtom = compAtom; H.atoms = atoms; H.aStart = aStart; H.aCon = aCon;
    H.rowStart = rowStart; H.col = col; H.conAtoms = conAtoms; H.dist = dist; H.redMass = redMass; H.val = val;
    H.distD = distD; H.redMassD = redMassD;
}

static void build_ccma(b200md_ctx* c) {
    const int nc = (int) c->ccmaCons.size();
    c->ccma = CcmaDev{};
    if (nc == 0) return;
    require(!c->p2p && c->world == 1, "general (CCMA) constraint networks are not supported in multi-GPU runs");
    const CcmaInput in{c->natoms, c->mass, c->ccmaCons, c->conI, c->conJ, c->conD, c->angles.atoms, c->angles.params};
    CcmaHost H;
    ccma_host_setup(&in, H);
    // ---- device ----
    c->ccCompCon.upload(H.compCon); c->ccCompAtom.upload(H.compAtom); c->ccConAtoms.upload(H.conAtoms); c->ccDist.upload(H.dist); c->ccRedMass.upload(H.redMass);
    c->ccRowStart.upload(H.rowStart); c->ccCol.upload(H.col); c->ccVal.upload(H.val); c->ccAtoms.upload(H.atoms); c->ccAStart.upload(H.aStart); c->ccACon.upload(H.aCon);
    c->ccRij.alloc(nc); c->ccDelta1.alloc(nc); c->ccDelta2.alloc(nc); c->ccXold.alloc(c->npad); c->ccXunc.alloc(c->npad);
    CcmaDev& cc = c->ccma;
    cc.ncomp = H.ncomp; cc.ncon = nc; cc.natomsC = (int) H.atoms.size();
    cc.compConStart = c->ccCompCon.p; cc.compAtomStart = c->ccCompAtom.p; cc.conAtoms = c->ccConAtoms.p; cc.conDist = c->ccDist.p; cc.conRedMass = c->ccRedMass.p;
    cc.rowStart = c->ccRowStart.p; cc.col = c->ccCol.p; cc.val = c->ccVal.p; cc.atoms = c->ccAtoms.p; cc.aStart = c->ccAStart.p; cc.aCon = c->ccACon.p;
    cc.rij = c->ccRij.p; cc.delta1 = c->ccDelta1.p; cc.delta2 = c->ccDelta2.p; cc.xold = c->ccXold.p; cc.xunc = c->ccXunc.p;
    cc.maxIter = 150;                   // ReferenceCCMAAlgorithm.cpp:55
    if (c->mixed()) {
        c->ccDistD.upload(H.distD); c->ccRedMassD.upload(H.redMassD);
        c->ccRijD.alloc(nc); c->ccDelta1D.alloc(nc); c->ccDelta2D.alloc(nc);
        c->ccXoldD.alloc(c->npad); c->ccXuncD.alloc(c->npad); c->ccXposD.alloc(c->npad);
        cc.conDistD = c->ccDistD.p; cc.conRedMassD = c->ccRedMassD.p;
        cc.rijD = c->ccRijD.p; cc.delta1D = c->ccDelta1D.p; cc.delta2D = c->ccDelta2D.p;
        cc.xoldD = c->ccXoldD.p; cc.xuncD = c->ccXuncD.p; cc.xposD = c->ccXposD.p;
    }
}

// CCMA host setup without a context or a device (tests): classification + approximate inverse of the coupling matrix.
// out_order[k] = index (into the caller's constraint arrays) of sorted constraint k; CSR in the SORTED numbering.
// Returns the number of non-zeros (or -1; -2 if cap is too small).
extern "C" int b200md_ccma_setup_probe(int natoms, const double* mass, int ncon, const int* p1, const int* p2, const double* dist,
                                       int nangles, const int* a1, const int* a2, const int* a3, const double* theta0,
                                       int* out_ncomp, int* out_nccma, int* out_order, int* row_start, int* col, float* val, int cap) {
    try {
        std::vector<double> m(mass, mass + natoms), cd(dist, dist + ncon);
        std::vector<int> ci(p1, p1 + ncon), cj(p2, p2 + ncon); std::vector<int4> aa(nangles); std::vector<double2> ap(nangles);
        for (int i = 0; i < nangles; i++) { aa[i] = make_int4(a1[i], a2[i], a3[i], 0); ap[i] = make_double2(theta0[i], 0.0); }
        std::vector<int4> ua; std::vector<int> ut; std::vector<float4> up; std::vector<int> ccmaCons;
        std::string err;
        if (!classify_units(natoms, m.data(), ci, cj, cd, ua, ut, up, err, &ccmaCons)) { g_create_error = err; return -1; }
        *out_nccma = (int) ccmaCons.size();
        *out_ncomp = 0;
        if (ccmaCons.empty()) { row_start[0] = 0; return 0; }
        const CcmaInput in{natoms, m, ccmaCons, ci, cj, cd, aa, ap};
        CcmaHost H;
        ccma_host_setup(&in, H);
        *out_ncomp = H.ncomp;
        if ((int) H.col.size() > cap) return -2;
        for (size_t k = 0; k < H.order.size(); k++) out_order[k] = ccmaCons[H.order[k]];
        for (size_t k = 0; k < H.rowStart.size(); k++) row_start[k] = H.rowStart[k];
        for (size_t k = 0; k < H.col.size(); k++) { col[k] = H.col[k]; val[k] = H.val[k]; }
        return (int) H.col.size();
    } catch (std::exception& e) { g_create_error = e.what(); return -1; }
}

// dry run of the constraint classification (no context, no device): 0 = every constraint is supported
extern "C" int b200md_check_constraints(int natoms, const double* mass, int n, const int* p1, const int* p2, const double* d, char* msg, int msglen) {
    try {
        std::vector<int> ci(p1, p1+n), cj(p2, p2+n); std::vector<double> cd(d, d+n);
        std::vector<int4> ua; std::vector<int> ut; std::vector<float4> up;
        std::string err;
        if (classify_units(natoms, mass, ci, cj, cd, ua, ut, up, err)) return 0;
        if (msg && msglen > 0) { strncpy(msg, err.c_str(), msglen-1); msg[msglen-1] = 0; }
        return -1;
    } catch (std::exception& e) { if (msg && msglen > 0) { strncpy(msg, e.what(), msglen-1); msg[msglen-1] = 0; } return -1; }
}

// B-spline moduli (pme_calculate_bsplines_moduli, ReferencePME.cpp:98-193)
static std::vector<double> bspline_moduli(int n) {
    const int order = B200MD_PME_ORDER;
    std::vector<double> data(order, 0.0), bs(std::max(n, order+1), 0.0), mod(n);
    data[order-1] = 0; data[1] = 0; data[0] = 1;
    for (int k = 3; k < order; k++) {
        double div = 1.0/(k-1.0);
        data[k-1] = 0;
        for (int l = 1; l < k-1; l++) data[k-l-1] = div*(l*data[k-l-2] + (k-l)*data[k-l-1]);
        data[0] = div*data[0];
    }
    double div = 1.0/(order-1);
    data[order-1] = 0;
    for (int l = 1; l < order-1; l++) data[order-l-1] = div*(l*data[order-l-2] + (order-l)*data[order-l-1]);
    data[0] = div*data[0];
    for (int i = 1; i <= order; i++) bs[i] = data[i-1];
    for (int i = 0; i < n; i++) {
        double sc = 0, ss = 0;
        for (int j = 0; j < n && j < (int) bs.size(); j++) {
            double arg = (2.0*M_PI*i*j)/n;
            sc += bs[j]*std::cos(arg); ss += bs[j]*std::sin(arg);
        }
        mod[i] = sc*sc + ss*ss;
    }
    for (int i = 0; i < n; i++)
        if (mod[i] < 1.0e-7) mod[i] = (mod[(i-1+n)%n] + mod[(i+1)%n])/2;
    return mod;
}

static void make_fft_plan(int n, FftPlanDev& plan, DevBuf<real2>& tw) {
    plan.n = n;
    if (!fft_make_radices(n, plan.radix, &plan.nstages))
        throw std::runtime_error("B200 platform: PME grid dimension " + std::to_string(n) + " has a prime factor > 13; choose a dimension that factors into radices <= 16");
    std::vector<real2> t(n);
    for (int k = 0; k < n; k++) { double a = -2.0*M_PI*k/n; t[k].x = (real) std::cos(a); t[k].y = (real) std::sin(a); }
    tw.upload(t);
    plan.tw = tw.p;
}

static void setup_pme(b200md_ctx* c, int nx, int ny, int nz, double alpha) {
    PmeDev& p = c->pme;
    p.nx = nx; p.ny = ny; p.nz = nz; p.nzc = nz/2 + 1; p.alpha = alpha;
    int dev = 0, maxSmem = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&maxSmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
    if (fft_plane_smem_bytes(ny, nz) > (size_t) maxSmem || fft_line_smem_bytes(nx) > (size_t) maxSmem)
        throw std::runtime_error("B200 platform: PME grid plane does not fit in shared memory (max about 160x160 per slab)");
    pme_brick_setup(maxSmem);
    c->brickPoints = std::min(c->brickPoints, (maxSmem - 1024)/(int) sizeof(long long));
    c->grid.alloc((size_t) nx*ny*nz);
    c->gridFixed.alloc((size_t) nx*ny*nz);
    p.gridFixed = c->gridFixed.p;
    c->cgrid.alloc((size_t) nx*ny*p.nzc);
    c->eterm.alloc((size_t) nx*ny*p.nzc);
    p.grid = c->grid.p; p.cgrid = c->cgrid.p; p.eterm = c->eterm.p;
    const int n[3] = {nx, ny, nz};
    for (int d = 0; d < 3; d++) {
        make_fft_plan(n[d], p.plan[d], c->tw[d]);
        c->moduli[d].upload(bspline_moduli(n[d]));
        p.moduli[d] = c->moduli[d].p;
    }
}


// ---------------------------------------------------------------- multi-GPU window (peer-memory data plane, comm.cu)
static size_t align_up(size_t x, size_t a) { return (x + a - 1)/a*a; }

// Lay the window out, allocate it, exchange the IPC handles (through the NCCL communicator that b200md_comm_init made: the
// only use of NCCL besides the rare energy reduction) and map every peer.  Called at the top of b200md_finalize; the state
// arrays that peers store into (posq, velm, force, the potential grid) are then carved out of the window.
static void setup_window(b200md_ctx* c) {
    const int P = c->world, NP = c->npad;
    require(P <= B200MD_MAX_RANKS, "at most 8 ranks");
    CommDev& cd = c->cd;
    cd = CommDev{};
    cd.rank = c->rank; cd.world = P;
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = align_up(off + bytes, 256); return o; };
    cd.offFlags = take((size_t) CH_COUNT*B200MD_MAX_RANKS*sizeof(unsigned long long));
    cd.offCm = take((size_t) B200MD_MAX_RANKS*12*sizeof(double));
    cd.offPosq = take((size_t) NP*sizeof(float4));
    cd.offVelm = take((size_t) NP*sizeof(float4));
    cd.offForce = take((size_t) 3*NP*sizeof(long long));
    cd.offFinbox = take((size_t) P*3*NP*sizeof(long long));
    const bool pme = c->haveNb && c->nbdesc.method == B200MD_NB_PME;
    if (pme) {
        const int nx = c->nbdesc.grid[0], ny = c->nbdesc.grid[1], nz = c->nbdesc.grid[2], nzc = nz/2 + 1;
        require(nx >= P, "PME grid has fewer x planes than ranks");
        const int plane = ny*nzc;
        cd.maxPlanes = 0;
        for (int q = 0; q <= P; q++) cd.xLo[q] = (int) ((long long) q*nx/P);
        for (int q = 0; q < P; q++) cd.maxPlanes = std::max(cd.maxPlanes, cd.xLo[q+1] - cd.xLo[q]);
        cd.lineChunk = (int) align_up((size_t) (plane + P - 1)/P, 16);
        cd.offGridInbox = take((size_t) P*cd.maxPlanes*ny*nz*sizeof(long long));
        cd.offLineBuf = take((size_t) nx*cd.lineChunk*sizeof(real2));
        cd.offPlaneBuf = take((size_t) cd.maxPlanes*plane*sizeof(real2));
        cd.offGrid = take((size_t) nx*ny*nz*sizeof(real));
    }
    c->windowBytes = off;
    CUDA_CHECK(cudaMalloc(&c->window, off));
    CUDA_CHECK(cudaMemset(c->window, 0, off));
    CUDA_CHECK(cudaDeviceSynchronize());            // nobody can map this window before the handle exchange below: it is zero when they do
    c->posq.attach(c->window + cd.offPosq, NP);
    c->velm.attach(c->window + cd.offVelm, NP);
    c->force.attach(c->window + cd.offForce, (size_t) 3*NP);
    if (pme) c->grid.attach(c->window + cd.offGrid, (size_t) c->nbdesc.grid[0]*c->nbdesc.grid[1]*c->nbdesc.grid[2]);
    // ---- handle exchange ----
    require(g_nccl.AllGather != nullptr, "libnccl lacks ncclAllGather");
    cudaIpcMemHandle_t mine;
    CUDA_CHECK(cudaIpcGetMemHandle(&mine, c->window));
    DevBuf<char> send, recv;
    send.alloc(sizeof(mine)); recv.alloc(sizeof(mine)*P);
    CUDA_CHECK(cudaMemcpy(send.p, &mine, sizeof(mine), cudaMemcpyHostToDevice));
    if (g_nccl.AllGather(send.p, recv.p, sizeof(mine), NCCL_INT8, c->comm, c->stream) != 0) throw std::runtime_error("ncclAllGather(ipc handles) failed");
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    std::vector<cudaIpcMemHandle_t> all(P);
    CUDA_CHECK(cudaMemcpy(all.data(), recv.p, sizeof(mine)*P, cudaMemcpyDeviceToHost));
    for (int q = 0; q < P; q++) {
        if (q == c->rank) { cd.peer[q] = c->window; continue; }
        cudaError_t e = cudaIpcOpenMemHandle(&c->peerMapped[q], all[q], cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess)
            throw std::runtime_error(std::string("cudaIpcOpenMemHandle(rank ") + std::to_string(q) + "): " + cudaGetErrorString(e) +
                                     " -- the peer-memory data plane needs CUDA IPC + P2P between the GPUs (B200MD_MGPU=nccl selects the NCCL all-reduce scheme)");
        cd.peer[q] = (char*) c->peerMapped[q];
    }
    c->commCounters.alloc(2); c->commCounters.zero();
    c->commDone.alloc(CH_COUNT); c->commDone.zero();
    cd.epoch = c->commCounters.p; cd.posNeed = c->commCounters.p + 1; cd.done = c->commDone.p;
    cd.posByPush = (pos_push_available() || P >= 8) ? 1 : 0;      // per-thread stores to 7 peers cost more than a kernel of bulk copies (k_integrate 40 us at 8 ranks)
}

// Ownership: rank q owns the integration units [unitLo[q], unitLo[q+1]) and with them the atoms [atomLo[q], atomLo[q+1]) --
// cuts are only made where the units before the cut hold exactly the atoms below some index (always the case for the usual
// molecule-by-molecule atom order).
// pure function (no device): the cuts for `P` ranks over `units` (sorted by first atom); atomLo / unitLo get P + 1 entries
static void ownership_cuts(const std::vector<int4>& units, int N, int P, int* atomLo, int* unitLo) {
    const int U = (int) units.size();
    std::vector<int> prefMax(U + 1, -1), sufMin(U + 1, N);
    auto lohi = [&](int u, int& lo, int& hi) {
        const int4 a = units[u]; const int v[4] = {a.x, a.y, a.z, a.w};
        lo = N; hi = -1;
        for (int k = 0; k < 4; k++) if (v[k] >= 0) { lo = std::min(lo, v[k]); hi = std::max(hi, v[k]); }
    };
    for (int u = 0; u < U; u++) { int lo, hi; lohi(u, lo, hi); prefMax[u+1] = std::max(prefMax[u], hi); }
    for (int u = U - 1; u >= 0; u--) { int lo, hi; lohi(u, lo, hi); sufMin[u] = std::min(sufMin[u+1], lo); }
    unitLo[0] = 0; atomLo[0] = 0; unitLo[P] = U; atomLo[P] = N;
    int u = 1;
    for (int q = 1; q < P; q++) {
        const long long target = (long long) q*N/P;
        // first valid cut at or after the target atom
        while (u < U && !(prefMax[u] < sufMin[u] && sufMin[u] >= target)) u++;
        require(u < U, "multi-GPU: cannot cut the atom range at integration-unit boundaries (molecules are not contiguous in atom order)");
        unitLo[q] = u; atomLo[q] = sufMin[u];
        u++;
    }
    for (int q = 0; q < P; q++) require(atomLo[q+1] > atomLo[q] && unitLo[q+1] > unitLo[q], "multi-GPU: a rank would own no atoms");
}
static void setup_ownership(b200md_ctx* c) {
    CommDev& cd = c->cd;
    ownership_cuts(c->hUnitAtoms, c->natoms, cd.world, cd.atomLo, cd.unitLo);
    cd.errFlag = c->counters.p + CT_OVERFLOW;
}
// the same without a context or a device (tests): constraints -> integration units -> cuts for `world` ranks
extern "C" int b200md_ownership_probe(int natoms, const double* mass, int ncon, const int* p1, const int* p2, const double* dist,
                                      int world, int* atom_lo, int* unit_lo) {
    try {
        if (world < 1 || world > B200MD_MAX_RANKS) return -1;
        std::vector<int> ci(p1, p1 + ncon), cj(p2, p2 + ncon); std::vector<double> cd(dist, dist + ncon);
        std::vector<int4> ua; std::vector<int> ut; std::vector<float4> up; std::vector<int> ccma;
        std::string err;
        if (!classify_units(natoms, mass, ci, cj, cd, ua, ut, up, err, &ccma)) { g_create_error = err; return -1; }
        ownership_cuts(ua, natoms, world, atom_lo, unit_lo);
        return (int) ua.size();
    } catch (std::exception& e) { g_create_error = e.what(); return -1; }
}

// ---------------------------------------------------------------- tile pools
// Capacity of ONE of the TILE_REGIONS slot pools.  The first guess assumes a homogeneous density; prepare_list() measures
// the pools after every list build that follows a change of the state from outside and grows them (slabs, droplets,
// vacuum around a solute and box changes are then handled instead of raising "capacity exceeded").
static int initial_pool_capacity(const b200md_ctx* c) {
    const int nbk = c->nblocks, N = c->natoms;
    const double rc = c->nbdesc.cutoff;
    // worst case (every block pair interacts): i-block ib emits at most nbk - ib + 2 tiles (its j-blocks, the diagonal
    // tile on its own, one partial tile); pool 0 holds the smallest ib and is the fullest
    double poolCap = 0;
    for (int ib = 0; ib < nbk; ib += TILE_REGIONS) poolCap += nbk - ib + 2;
    if (c->nb.method != B200MD_NB_NOCUTOFF && c->haveBox) {
        const double vol = c->boxA[0]*c->boxB[1]*c->boxC[2];
        const double rp = rc*(1.0 + c->padFrac);
        const double pairs = 0.5*N*(N/vol)*(4.0/3.0*M_PI*rp*rp*rp);
        const double est = pairs/(1024.0*0.15) + 18.0*nbk;           // tiles at >= 15 % fill + partial tiles
        poolCap = std::min(poolCap, 1.25*est/TILE_REGIONS + 64);     // + slack for the imbalance between pools
    }
    poolCap = std::min(poolCap, 16.0e6/TILE_REGIONS);
    if (c->pmeOnly) poolCap = 1;
    return (int) poolCap + 1;
}
static int worst_pool_capacity(const b200md_ctx* c) {
    double cap = 0;
    for (int ib = 0; ib < c->nblocks; ib += TILE_REGIONS) cap += c->nblocks - ib + 2;
    return (int) std::min(cap, 2.0e9/TILE_REGIONS/32) + 1;
}
static void alloc_tile_pools(b200md_ctx* c, int poolCap) {
    NbDev& nb = c->nb;
    nb.maxTiles = poolCap*TILE_REGIONS;
    for (int l = 0; l < 2; l++) { c->lists[l].alloc_tiles(nb.maxTiles); c->lists[l].bind(nb.list[l], c->listCounters.p + LC_STRIDE*l); }
}

// The reciprocal-space chain runs beside a tile kernel that holds every SM: one GPU, two streams, no SM partition.  Its FFT
// then runs as small CTAs that fit the slots retiring tile CTAs hand back (fft.cu); everywhere else it keeps the larger ones.
static bool fft_beside_tiles(const b200md_ctx* c) {
    return c->world == 1 && !c->pmeOnly && c->overlapPme && !c->nb.smPartition && c->nbdesc.method == B200MD_NB_PME;
}

// finalize: the custom torsions in the layout of k_custom_torsion (CustomTorsionDev): grouped by expression, each group padded
// to whole warps, and the programs, checked once more now that the number of global slots is final
static void upload_custom_torsions(b200md_ctx* c) {
    CustomTorsionTable& t = c->custom;
    CustomTorsionDev& d = c->ctd;
    d = CustomTorsionDev{};
    d.groupMask = 0xffffffffu;
    // the global values get their buffer even without terms: a CustomTorsionForce with no torsions may still name globals, and
    // b200md_set_custom_globals copies into this buffer after finalize
    t.globalsDev.alloc(std::max<size_t>(t.globals.size(), 1)); t.globalsDev.upload(t.globals);
    d.globals = t.globalsDev.p;
    if (t.n == 0) return;
    require(c->world == 1, "custom torsions are not supported in multi-GPU runs");
    require(t.group.empty() || (int) t.group.size() == t.n, "set_bonded_groups: group array length differs from the number of terms");
    for (int q = 0; q < 2*t.nprog; q++) {
        const char* why = custom_check_program(t.code.data(), t.progStart[q], t.progStart[q+1], t.stride, (int) t.globals.size());
        if (why) throw std::runtime_error(std::string(why) + " (program " + std::to_string(q) + ")");
    }
    t.slot.assign(t.n, 0);
    int cursor = 0;
    for (int p = 0; p < t.nprog; p++) {
        for (int i = 0; i < t.n; i++) if (t.prog[i] == p) t.slot[i] = cursor++;
        cursor = (cursor + 31)/32*32;
    }
    t.nslots = cursor;
    std::vector<int4> atoms(cursor, make_int4(0, 0, 0, 0));
    std::vector<unsigned char> group(cursor, 0);
    std::vector<int> prog(cursor, -1);
    for (int i = 0; i < t.n; i++) { atoms[t.slot[i]] = t.atoms[i]; group[t.slot[i]] = t.group.empty() ? 0 : t.group[i]; prog[t.slot[i]] = t.prog[i]; }
    t.atomsDev.upload(atoms); t.groupDev.upload(group); t.progDev.upload(prog);
    const std::vector<double> par = t.slot_params();
    t.paramsDev.alloc(std::max<size_t>(par.size(), 1)); t.paramsDev.upload(par);
    t.codeDev.upload(t.code); t.immDev.upload(t.imm); t.progStartDev.upload(t.progStart);
    d.nslots = t.nslots; d.paramStride = t.stride;
    d.atoms = t.atomsDev.p; d.params = t.paramsDev.p; d.group = t.groupDev.p; d.prog = t.progDev.p;
    d.code = t.codeDev.p; d.imm = t.immDev.p; d.progStart = t.progStartDev.p;
}

extern "C" int b200md_finalize(b200md_ctx* ctx) {
    API_BEGIN(ctx)
    require(!ctx->finalized, "finalize called twice");
    b200md_ctx* c = ctx;
    const int N = c->natoms, NP = c->npad;
    if (!c->haveNb) { c->nbdesc = b200md_nonbonded_desc{}; c->nbdesc.method = B200MD_NB_NOCUTOFF; }
    NbDev& nb = c->nb;
    nb.natoms = N; nb.npad = NP; nb.nblocks = c->nblocks;
    nb.method = c->nbdesc.method;
    nb.rank = c->rank; nb.world = c->world;
    c->cd = CommDev{}; c->cd.world = 1;
    c->p2p = c->world > 1 && c->comm && !(getenv("B200MD_MGPU") && std::string(getenv("B200MD_MGPU")) == "nccl");
    if (c->p2p) setup_window(c);
    { const double cc = getenv("B200MD_CLOSE_NM") ? atof(getenv("B200MD_CLOSE_NM")) : 0.36; nb.closeCut2 = (float) (cc*cc); }
    // SM partition between the tile kernel and the reciprocal-space chain (B200MD_PME_SMS=k reserves k SMs; 0 = off)
    for (int w = 0; w < 4; w++) nb.pmeSmMask[w] = 0ull;
    nb.smPartition = false;
    // Off on one GPU (measured: the chain is latency bound and needs most SMs to be short, profiles/r02_sm_partition.md).
    // Multi-GPU (peer-memory data plane): the chain is a sequence of kernels that wait for the other ranks, and behind a tile
    // kernel that holds every SM it would only start when that has drained; here the default reserves as many SMs as the rank
    // has x planes (one slab CTA each), between 16 and 48.
    if (c->nbdesc.method == B200MD_NB_PME && !c->pmeOnly && c->overlapPme) {
        int want = 0;
        // at least one SM per x plane of this rank; the more ranks, the shorter the tile kernel and the longer (relatively)
        // the chain of exchanges: 44 / 40 / 64 SMs at 2 / 4 / 8 ranks for an 88^3 grid
        if (c->p2p) want = std::min(74, std::max((c->nbdesc.grid[0] + c->world - 1)/c->world, 16 + 6*c->world));
        if (getenv("B200MD_PME_SMS")) want = atoi(getenv("B200MD_PME_SMS"));
        const int got = want > 0 ? choose_pme_sms(want, nb.pmeSmMask) : 0;
        if (got > 0) {
            nb.smPartition = true;
            const int planes = (c->nbdesc.grid[0] + c->world - 1)/c->world;
            fft_set_compact(planes > got ? 2 : 1);
        }
    }
    // ---- state arrays ----
    c->posq.alloc(NP); c->posq.zero(); c->velm.alloc(NP);
    c->refPos.alloc(NP); c->refPos.zero(); c->atomShift.alloc(NP); c->sigeps.alloc(NP);
    c->listCounters.alloc(2*LC_STRIDE); c->listCounters.zero();
    for (int l = 0; l < 2; l++) c->lists[l].alloc(NP, c->nblocks);      // bound to nb.list[l] with the tile pools (alloc_tile_pools)
    c->force.alloc((size_t) 3*NP); c->force.zero(); c->forceS.alloc((size_t) 3*NP); c->forceS.zero();
    c->energy.alloc(B200MD_NUM_ENERGY); c->energy.zero(); c->cmScratch.alloc(12); c->cmScratch.zero();
    c->blocksDone.alloc(1); c->blocksDone.zero();
    c->sortedOf.alloc(NP); c->atomCell.alloc(NP); c->tmpSorted.alloc(NP);
    c->counters.alloc(16); c->counters.zero();
    c->stepCounter.alloc(1); c->stepCounter.zero();
    upload_velocities(c, c->velm.p, nullptr);        // in a mixed context too: nothing reads it there, but nothing is left uninitialised
    nb.posqCorr = nullptr; nb.velmD = nullptr;
    if (c->mixed()) {
        c->posqCorr.alloc(NP); c->posqCorr.zero(); c->velmD.alloc(NP); upload_velocities(c, c->velmD.p, nullptr);
        nb.posqCorr = c->posqCorr.p; nb.velmD = c->velmD.p;
    }
    nb.posq = c->posq.p; nb.velm = c->velm.p; nb.sigeps = c->sigeps.p; nb.force = c->force.p; nb.forceS = c->forceS.p; nb.energy = c->energy.p;
    nb.sortedOf = c->sortedOf.p;
    nb.refPos = c->refPos.p; nb.atomCell = c->atomCell.p; nb.tmpSorted = c->tmpSorted.p; nb.atomShift = c->atomShift.p;
    nb.counters = c->counters.p;
    // ---- cutoffs ----
    const double rc = c->nbdesc.cutoff;
    if (nb.method == B200MD_NB_NOCUTOFF) {
        nb.cutoff = 1e18f; nb.cutoff2 = 3e38f; nb.paddedCutoff2 = 3e38f; nb.halfPad2 = 3e38f;
    }
    else {
        const double pad = c->padFrac*rc;
        nb.cutoff = (float) rc; nb.cutoff2 = (float) (rc*rc); nb.paddedCutoff2 = (float) ((rc+pad)*(rc+pad)); nb.halfPad2 = (float) (0.25*pad*pad);
    }
    nb.useSwitch = c->nbdesc.use_switch; nb.switchDist = (float) c->nbdesc.switch_distance;
    nb.alpha = (float) c->nbdesc.ewald_alpha;
    if (nb.method == B200MD_NB_CUTOFF_PERIODIC || nb.method == B200MD_NB_CUTOFF_NONPERIODIC) {
        const double eps = c->nbdesc.rf_dielectric;
        nb.krf = (float) (std::pow(rc, -3.0)*(eps-1.0)/(2.0*eps+1.0));
        nb.crf = (float) ((1.0/rc)*(3.0*eps)/(2.0*eps+1.0));
    }
    // ---- exclusions (every exception is an exclusion) ----
    {
        std::vector<std::vector<int> > ex(N);
        for (const int2& a : c->exc.atoms) { ex[a.x].push_back(a.y); ex[a.y].push_back(a.x); }
        std::vector<int> start(N+1, 0), list;
        for (int i = 0; i < N; i++) {
            std::sort(ex[i].begin(), ex[i].end());
            ex[i].erase(std::unique(ex[i].begin(), ex[i].end()), ex[i].end());
            start[i+1] = start[i] + (int) ex[i].size();
            list.insert(list.end(), ex[i].begin(), ex[i].end());
        }
        if (list.empty()) list.push_back(0);
        c->exclStart.upload(start); c->exclList.upload(list);
        nb.exclStart = c->exclStart.p; nb.exclList = c->exclList.p;
    }
    // ---- tile capacity: TILE_REGIONS equal slot pools, i-block ib allocates from pool ib % TILE_REGIONS (flush_tile) ----
    alloc_tile_pools(c, initial_pool_capacity(c));
    // ---- bonded (exceptions: upload_params) ----
    BondedDev& bd = c->bd;
    c->bonds.upload(bd.nbonds, bd.bondAtoms, bd.bondParams, bd.bondGroup);
    c->angles.upload(bd.nangles, bd.angleAtoms, bd.angleParams, bd.angleGroup);
    c->torsions.upload(bd.ntorsions, bd.torsionAtoms, bd.torsionParams, bd.torsionGroup);
    c->rb.upload(bd.nrb, bd.rbAtoms, bd.rbParams, bd.rbGroup);
    c->cmap.upload(bd.ncmap, bd.cmapAtoms, bd.cmapCoeff, bd.cmapGroup);
    c->cmap.mapDev.upload(c->cmap.map); c->cmap.mapsDev.upload(c->cmap.maps); bd.cmapMap = c->cmap.mapDev.p; bd.cmapMaps = c->cmap.mapsDev.p;
    bd.excPeriodic = c->nbdesc.exceptions_periodic;
    bd.groupMask = 0xffffffffu;
    upload_custom_torsions(c);
    upload_params(c);
    build_units(c);
    build_ccma(c);
    if (c->p2p) {
        setup_ownership(c);
        if (nb.method == B200MD_NB_PME) {
            PmeDev probe{}; probe.nx = c->nbdesc.grid[0]; probe.ny = c->nbdesc.grid[1]; probe.nz = c->nbdesc.grid[2]; probe.nzc = probe.nz/2 + 1;
            require(fft_slab_path(probe), "multi-GPU: the PME grid plane does not fit the slab FFT kernels (B200MD_MGPU=nccl selects the NCCL scheme)");
        }
    }
    // ---- molecules (connected components of bonds, angles, torsions, RB torsions, CMAP terms, custom torsions, constraints and exceptions) for the wrap at list
    // builds; off for non-periodic systems and with more than one rank (every rank would have to wrap in the same step,
    // and the reciprocal-space rank builds no list) ----
    c->cellOffset.alloc((size_t) 3*NP); c->cellOffset.zero();
    nb.cellOffset = c->cellOffset.p; nb.nmol = 0; nb.molStart = nullptr; nb.molAtoms = nullptr;
    if ((nb.method == B200MD_NB_CUTOFF_PERIODIC || nb.method == B200MD_NB_PME) && c->world == 1 && !c->pmeOnly) {
        std::vector<int> parent(N);
        for (int i = 0; i < N; i++) parent[i] = i;
        auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
        auto join = [&](int a, int b) { a = find(a); b = find(b); if (a != b) parent[std::max(a, b)] = std::min(a, b); };
        for (const int2& a : c->bonds.atoms) join(a.x, a.y);
        for (const int4& a : c->angles.atoms) { join(a.x, a.y); join(a.y, a.z); }
        for (auto* t : {&c->torsions.atoms, &c->rb.atoms, &c->cmap.atoms, &c->custom.atoms}) for (const int4& a : *t) { join(a.x, a.y); join(a.y, a.z); join(a.z, a.w); }
        for (size_t d = 1; d < c->cmap.atoms.size(); d += 2) join(c->cmap.atoms[d-1].x, c->cmap.atoms[d].x);     // a CMAP term's two dihedrals
        for (size_t i = 0; i < c->conI.size(); i++) join(c->conI[i], c->conJ[i]);
        for (const int2& a : c->exc.atoms) join(a.x, a.y);
        std::vector<int> molOf(N), count;
        std::map<int, int> id;
        for (int i = 0; i < N; i++) {
            const int r = find(i);
            auto it = id.find(r);
            if (it == id.end()) { it = id.insert(std::make_pair(r, (int) count.size())).first; count.push_back(0); }
            molOf[i] = it->second; count[it->second]++;
        }
        std::vector<int> start(count.size() + 1, 0), fill(count.size(), 0), atoms(N);
        for (size_t m = 0; m < count.size(); m++) start[m+1] = start[m] + count[m];
        for (int i = 0; i < N; i++) atoms[start[molOf[i]] + fill[molOf[i]]++] = i;      // ascending inside a molecule: the first atom is its anchor
        c->molStart.upload(start); c->molAtoms.upload(atoms);
        nb.nmol = (int) count.size(); nb.molStart = c->molStart.p; nb.molAtoms = c->molAtoms.p;
    }
    if (nb.method == B200MD_NB_PME) setup_pme(c, c->nbdesc.grid[0], c->nbdesc.grid[1], c->nbdesc.grid[2], c->nbdesc.ewald_alpha);
    // the chain's CTAs join SMs that run the tile kernel (the brick's static shared memory is a few words)
    if (fft_beside_tiles(c)) pair_set_carveout(fft_cta_smem_bytes(c->pme), sizeof(long long)*(size_t) c->brickPoints + 64);
    c->finalized = true;
    try { apply_box(c); } catch (...) { c->finalized = false; throw; }      // e.g. box smaller than twice the cutoff: the caller may fix the box and finalize again
    c->integ.stepCounter = c->stepCounter.p;
    c->integ.fused = 0; c->integ.cmEveryStep = 0; c->integ.cmScratch = c->cmScratch.p; c->integ.blocksDone = c->blocksDone.p;
    API_END(ctx)
}

extern "C" int b200md_update_nonbonded_params(b200md_ctx* ctx, const double* q, const double* sig, const double* eps,
                                              int nexc, const double* eqq, const double* esig, const double* eeps, double dispCoef) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update params before finalize");
    require(nexc == (int) ctx->exc.atoms.size(), "update_nonbonded_params: the number of exceptions cannot change");
    ctx->charge.assign(q, q + ctx->natoms); ctx->sigma.assign(sig, sig + ctx->natoms); ctx->epsilon.assign(eps, eps + ctx->natoms);
    for (int e = 0; e < nexc; e++) ctx->exc.params[e] = make_double3(eqq[e], esig[e], eeps[e]);
    ctx->dispersionCoefficient = dispCoef;
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    upload_params(ctx);
    request_rebuild(ctx);         // the list holds sorted copies of the parameters
    invalidate_graph(ctx);
    API_END(ctx)
}

// Calc{HarmonicBond,HarmonicAngle,PeriodicTorsion}ForceKernel::copyParametersToContext (kernels.h:305,375,445):
// same topology, new parameters.  kind: B200MD_BONDED_BONDS (a=length,b=k), _ANGLES (a=angle,b=k), _TORSIONS (a=phase,b=k,per)
extern "C" int b200md_update_bonded_params(b200md_ctx* ctx, int kind, int n, const double* a, const double* b, const int* periodicity) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_bonded_params before finalize");
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    if (kind == B200MD_BONDED_BONDS) {
        require(n == ctx->bonds.n, "the number of bonds cannot change");
        for (int i = 0; i < n; i++) ctx->bonds.params[i] = make_double2(a[i], b[i]);
        ctx->bonds.paramsDev.upload(ctx->bonds.params);
    }
    else if (kind == B200MD_BONDED_ANGLES) {
        require(n == ctx->angles.n, "the number of angles cannot change");
        for (int i = 0; i < n; i++) ctx->angles.params[i] = make_double2(a[i], b[i]);
        ctx->angles.paramsDev.upload(ctx->angles.params);
    }
    else if (kind == B200MD_BONDED_TORSIONS) {
        require(n == ctx->torsions.n, "the number of torsions cannot change");
        for (int i = 0; i < n; i++) ctx->torsions.params[i] = make_double4(b[i], a[i], (double) periodicity[i], 0);
        ctx->torsions.paramsDev.upload(ctx->torsions.params);
    }
    else throw std::runtime_error("unknown bonded kind");
    API_END(ctx)
}

// Calc{RBTorsion,CMAPTorsion}ForceKernel::copyParametersToContext (kernels.h:480, 515): the device arrays keep their size,
// so they are overwritten in place and captured step graphs stay valid.
extern "C" int b200md_update_rb_torsion_params(b200md_ctx* ctx, int n, const double* c) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_rb_torsion_params before finalize");
    require(n == ctx->rb.n, "updateParametersInContext: The number of torsions has changed");
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->rb.params.assign(c, c + 6*(size_t) n);
    ctx->rb.paramsDev.upload(ctx->rb.params);
    API_END(ctx)
}
extern "C" int b200md_update_cmap_params(b200md_ctx* ctx, int nmaps, const int* size, const double* coeff, int n, const int* map) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_cmap_params before finalize");
    require(nmaps == (int) ctx->cmap.maps.size(), "updateParametersInContext: The number of maps has changed");
    require(n == ctx->cmap.n, "updateParametersInContext: The number of CMAP torsions has changed");
    for (int m = 0; m < nmaps; m++) require(size[m] == ctx->cmap.maps[m].y, "updateParametersInContext: The size of a map has changed");
    for (int i = 0; i < n; i++) require(map[i] >= 0 && map[i] < nmaps, "CMAP torsion: map index out of range");
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->cmap.params.assign(coeff, coeff + ctx->cmap.params.size());
    ctx->cmap.map.assign(map, map + n);
    ctx->cmap.paramsDev.upload(ctx->cmap.params); ctx->cmap.mapDev.upload(ctx->cmap.map);
    API_END(ctx)
}

// CalcCustomTorsionForceKernel::copyParametersToContext (kernels.h:544): same terms and programs, new parameters, into the
// same device buffer.
extern "C" int b200md_update_custom_torsion_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_custom_torsion_params before finalize");
    CustomTorsionTable& t = ctx->custom;
    require(n == t.n, "updateParametersInContext: The number of torsions has changed");
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    t.params.assign(params, params + (size_t) n*t.stride);
    if (n) t.paramsDev.upload(t.slot_params());
    API_END(ctx)
}

// ---------------------------------------------------------------- state
// Multi-GPU (peer-memory data plane): only the owner integrates an atom.  Positions reach every rank with the step itself;
// velocities stay with the owner until somebody reads them from the host side.
static void sync_positions(b200md_ctx* c) { if (c->p2p && c->finalized) launch_pos_wait(c->nb, c->cd, c->stream); }
static void sync_velocities(b200md_ctx* c) {
    if (!c->p2p || !c->velStale) return;
    launch_vel_push(c->nb, c->cd, c->stream);
    c->kernelLaunches += 2;
    c->velStale = false;
}
static void host_set_state(b200md_ctx* c) {       // the host wrote the full state on every rank: nothing to wait for
    if (!c->p2p) return;
    const unsigned long long zero = 0ull;
    CUDA_CHECK(cudaMemcpyAsync(c->cd.posNeed, &zero, sizeof(zero), cudaMemcpyHostToDevice, c->stream));
}

extern "C" int b200md_set_positions(b200md_ctx* ctx, const double* x) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    require(ctx->finalized, "set_positions before finalize");
    const int N = ctx->natoms;
    const double sk = std::sqrt(B200MD_ONE_4PI_EPS0);
    ctx->hbuf4.resize(ctx->npad);
    for (int i = 0; i < N; i++) ctx->hbuf4[i] = make_float4((float) x[3*i], (float) x[3*i+1], (float) x[3*i+2], (float) (ctx->charge[i]*sk));
    for (int i = N; i < ctx->npad; i++) ctx->hbuf4[i] = make_float4(0, 0, 0, 0);
    if (!ctx->haveOrigin) {
        // primary-cell origin = lower corner of the structure (first call only; later calls keep it so that the step
        // graph's kernel parameters stay valid)
        double lo[3] = {1e300, 1e300, 1e300};
        for (int i = 0; i < N; i++) for (int k = 0; k < 3; k++) lo[k] = std::min(lo[k], x[3*i+k]);
        for (int k = 0; k < 3; k++) ctx->nb.origin[k] = std::isfinite(lo[k]) ? lo[k] : 0.0;
        ctx->haveOrigin = true;
        invalidate_graph(ctx);
    }
    sync_positions(ctx);          // the peers' stores of the last step must not land after this upload
    CUDA_CHECK(cudaMemcpyAsync(ctx->posq.p, ctx->hbuf4.data(), sizeof(float4)*ctx->npad, cudaMemcpyHostToDevice, ctx->stream));
    if (ctx->mixed()) {           // low parts (engine.h: pos_split)
        ctx->hcorr4.assign(ctx->npad, make_float4(0, 0, 0, 0));
        for (int i = 0; i < N; i++) {
            float hi; float4& l = ctx->hcorr4[i];       // hi: as uploaded to posq above
            pos_split(x[3*i], hi, l.x); pos_split(x[3*i+1], hi, l.y); pos_split(x[3*i+2], hi, l.z);
        }
        CUDA_CHECK(cudaMemcpyAsync(ctx->posqCorr.p, ctx->hcorr4.data(), sizeof(float4)*ctx->npad, cudaMemcpyHostToDevice, ctx->stream));
    }
    host_set_state(ctx);
    CUDA_CHECK(cudaMemsetAsync(ctx->cellOffset.p, 0, sizeof(int)*3*ctx->npad, ctx->stream));
    request_rebuild(ctx);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    API_END(ctx)
}
extern "C" int b200md_get_positions(b200md_ctx* ctx, double* x) {
    API_BEGIN(ctx)
    ctx->hbuf4.resize(ctx->npad);
    sync_positions(ctx);
    CUDA_CHECK(cudaMemcpyAsync(ctx->hbuf4.data(), ctx->posq.p, sizeof(float4)*ctx->npad, cudaMemcpyDeviceToHost, ctx->stream));
    if (ctx->mixed()) {
        ctx->hcorr4.resize(ctx->npad);
        CUDA_CHECK(cudaMemcpyAsync(ctx->hcorr4.data(), ctx->posqCorr.p, sizeof(float4)*ctx->npad, cudaMemcpyDeviceToHost, ctx->stream));
    }
    check_flags(ctx);
    for (int i = 0; i < ctx->natoms; i++) { x[3*i] = ctx->hbuf4[i].x; x[3*i+1] = ctx->hbuf4[i].y; x[3*i+2] = ctx->hbuf4[i].z; }
    if (ctx->mixed())
        for (int i = 0; i < ctx->natoms; i++) {
            const float4 h = ctx->hbuf4[i], l = ctx->hcorr4[i];
            x[3*i] = pos_join(h.x, l.x); x[3*i+1] = pos_join(h.y, l.y); x[3*i+2] = pos_join(h.z, l.z);
        }
    if (ctx->nb.nmol > 0) {
        // undo the internal molecule wrapping: the caller sees the continuous trajectory, like the Reference platform's
        const int NP = ctx->npad;
        ctx->hoffset.resize((size_t) 3*NP);
        CUDA_CHECK(cudaMemcpy(ctx->hoffset.data(), ctx->cellOffset.p, sizeof(int)*3*NP, cudaMemcpyDeviceToHost));
        for (int i = 0; i < ctx->natoms; i++) {
            const int kx = ctx->hoffset[i], ky = ctx->hoffset[i + NP], kz = ctx->hoffset[i + 2*NP];
            if (kx | ky | kz) {
                x[3*i]   += kx*ctx->boxA[0] + ky*ctx->boxB[0] + kz*ctx->boxC[0];
                x[3*i+1] += ky*ctx->boxB[1] + kz*ctx->boxC[1];
                x[3*i+2] += kz*ctx->boxC[2];
            }
        }
    }
    API_END(ctx)
}
extern "C" int b200md_set_velocities(b200md_ctx* ctx, const double* v) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    require(ctx->finalized, "set_velocities before finalize");
    if (ctx->mixed()) upload_velocities(ctx, ctx->velmD.p, v);
    else upload_velocities(ctx, ctx->velm.p, v);
    ctx->velStale = false;
    API_END(ctx)
}
extern "C" int b200md_get_velocities(b200md_ctx* ctx, double* v) {
    API_BEGIN(ctx)
    ctx->hbuf4.resize(ctx->npad);
    sync_velocities(ctx);
    if (ctx->mixed()) {
        std::vector<double4> vd(ctx->npad);
        CUDA_CHECK(cudaMemcpyAsync(vd.data(), ctx->velmD.p, sizeof(double4)*ctx->npad, cudaMemcpyDeviceToHost, ctx->stream));
        check_flags(ctx);
        for (int i = 0; i < ctx->natoms; i++) { v[3*i] = vd[i].x; v[3*i+1] = vd[i].y; v[3*i+2] = vd[i].z; }
    }
    else {
        CUDA_CHECK(cudaMemcpyAsync(ctx->hbuf4.data(), ctx->velm.p, sizeof(float4)*ctx->npad, cudaMemcpyDeviceToHost, ctx->stream));
        check_flags(ctx);
        for (int i = 0; i < ctx->natoms; i++) { v[3*i] = ctx->hbuf4[i].x; v[3*i+1] = ctx->hbuf4[i].y; v[3*i+2] = ctx->hbuf4[i].z; }
    }
    API_END(ctx)
}
extern "C" int b200md_get_forces(b200md_ctx* ctx, double* f) {
    API_BEGIN(ctx)
    ctx->hforce.resize((size_t) 3*ctx->npad);
    CUDA_CHECK(cudaMemcpyAsync(ctx->hforce.data(), ctx->force.p, sizeof(long long)*3*ctx->npad, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    const double s = 1.0/B200MD_FORCE_SCALE;
    for (int i = 0; i < ctx->natoms; i++)
        for (int k = 0; k < 3; k++) f[3*i+k] = s*(double) ctx->hforce[(size_t) k*ctx->npad + i];
    API_END(ctx)
}
extern "C" int b200md_set_time(b200md_ctx* ctx, double t) { if (!ctx) return -1; ctx->time = t; return 0; }
extern "C" double b200md_get_time(b200md_ctx* ctx) { return ctx ? ctx->time : 0.0; }
extern "C" int64_t b200md_get_step_count(b200md_ctx* ctx) { return ctx ? ctx->stepCount : 0; }
extern "C" void* b200md_cuda_stream(b200md_ctx* ctx) { return ctx ? (void*) ctx->stream : nullptr; }
extern "C" int b200md_synchronize(b200md_ctx* ctx) {
    API_BEGIN(ctx)
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    check_flags(ctx);
    API_END(ctx)
}

// ---------------------------------------------------------------- checkpoint
// Header, then state_spans: version 2 (single precision) posq | velm | cellOffset, version 3 (mixed precision) posq | posqCorr
// | velmD | cellOffset.  cellOffset stays last in both.  A blob is only loaded into a context of its own precision.
struct CkptHeader { char magic[8]; int version; int natoms; double time; int64_t stepCount; double box[9]; unsigned long long rngStep; };
static int ckpt_version(const b200md_ctx* c) { return c->mixed() ? 3 : 2; }
static int64_t ckpt_bytes(const b200md_ctx* c) {
    int64_t n = sizeof(CkptHeader);
    for (const DevSpan& s : state_spans(c)) n += s.bytes;
    return n;
}
extern "C" int64_t b200md_checkpoint_save(b200md_ctx* ctx, void* buf, int64_t cap) {
    if (!ctx) return -1;
    const int64_t need = ckpt_bytes(ctx);
    if (!buf) return need;
    try {
        CUDA_CHECK(cudaSetDevice(ctx->device));
        require(cap >= need, "checkpoint buffer too small");
        sync_positions(ctx); sync_velocities(ctx);
        CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
        CkptHeader h; memset(&h, 0, sizeof(h));
        memcpy(h.magic, "B200MDCK", 8); h.version = ckpt_version(ctx); h.natoms = ctx->natoms; h.time = ctx->time; h.stepCount = ctx->stepCount;
        for (int i = 0; i < 3; i++) { h.box[i] = ctx->boxA[i]; h.box[3+i] = ctx->boxB[i]; h.box[6+i] = ctx->boxC[i]; }
        CUDA_CHECK(cudaMemcpy(&h.rngStep, ctx->stepCounter.p, sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        char* p = (char*) buf;
        memcpy(p, &h, sizeof(h)); p += sizeof(h);
        for (const DevSpan& s : state_spans(ctx)) { CUDA_CHECK(cudaMemcpy(p, s.p, s.bytes, cudaMemcpyDeviceToHost)); p += s.bytes; }
        return need;
    } catch (std::exception& e) { ctx->err = e.what(); return -1; }
}
extern "C" int b200md_checkpoint_load(b200md_ctx* ctx, const void* buf, int64_t size) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    require(ctx->finalized, "checkpoint_load before finalize");
    require(size >= (int64_t) sizeof(CkptHeader), "checkpoint blob too small");
    CkptHeader h; memcpy(&h, buf, sizeof(h));
    require(memcmp(h.magic, "B200MDCK", 8) == 0 && (h.version == 2 || h.version == 3) && h.natoms == ctx->natoms, "checkpoint blob does not match this context");
    require(h.version == ckpt_version(ctx), h.version == 3 ? "the checkpoint was written in mixed precision and this context is single precision"
                                                           : "the checkpoint was written in single precision and this context is mixed precision");
    require(size >= ckpt_bytes(ctx), "checkpoint blob too small");
    sync_positions(ctx);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    ctx->time = h.time; ctx->stepCount = h.stepCount;
    for (int i = 0; i < 3; i++) { ctx->boxA[i] = h.box[i]; ctx->boxB[i] = h.box[3+i]; ctx->boxC[i] = h.box[6+i]; }
    const char* p = (const char*) buf + sizeof(h);
    for (const DevSpan& s : state_spans(ctx)) { CUDA_CHECK(cudaMemcpy(s.p, p, s.bytes, cudaMemcpyHostToDevice)); p += s.bytes; }
    CUDA_CHECK(cudaMemcpy(ctx->stepCounter.p, &h.rngStep, sizeof(unsigned long long), cudaMemcpyHostToDevice));
    host_set_state(ctx); ctx->velStale = false;
    if (ctx->haveBox) apply_box(ctx);
    request_rebuild(ctx);
    API_END(ctx)
}

// Multi-GPU role split (replicated atoms): with PME and world > 1 the LAST rank computes reciprocal space for all atoms and
// nothing else; the other world-1 ranks share the direct-space tiles (by i-block: list construction AND tile kernel) and the
// bonded terms.  Returns the rank's view of the sharding.
static bool role_split(const b200md_ctx* c) { return c->world > 1 && c->comm && !c->p2p && c->nb.method == B200MD_NB_PME && c->haveNb; }
static NbDev role_nb(const b200md_ctx* c) {
    NbDev nb = c->nb;
    if (role_split(c)) {
        if (c->rank == c->world - 1) { nb.rank = 0; nb.world = 1; }
        else nb.world = c->world - 1;
    }
    return nb;
}

// ---------------------------------------------------------------- force evaluation
// PME parameters of the next spread launch: the brick path needs a list that covers every atom on this GPU
static PmeDev pme_for_launch(const b200md_ctx* c) {
    PmeDev p = c->pme;
    p.brickAtoms = (c->pmeBrick && c->world == 1 && !c->pmeOnly && c->listBuilt) ? c->brickAtoms : 0;
    p.brickPoints = c->brickPoints;
    return p;
}

// Enqueue one force evaluation on the stream (no host sync).  Returns the number of kernels launched.
static int enqueue_forces(b200md_ctx* c, int terms, bool energy, bool forcesAlreadyZero = false, bool inStep = false, unsigned int groupMask = 0xffffffffu) {
    int launches = 0;
    cudaStream_t s = c->stream;
    if (!forcesAlreadyZero) CUDA_CHECK(cudaMemsetAsync(c->force.p, 0, sizeof(long long)*3*c->npad, s));
    if (energy) CUDA_CHECK(cudaMemsetAsync(c->energy.p, 0, sizeof(double)*B200MD_NUM_ENERGY, s));
    bool direct = (terms & B200MD_TERM_NB_DIRECT) && c->haveNb;
    bool recip = (terms & B200MD_TERM_NB_RECIP) && c->haveNb && c->nb.method == B200MD_NB_PME;
    // Multi-GPU role split (replicated atoms): the LAST rank computes reciprocal space for all atoms and nothing else; the
    // other world-1 ranks share the direct-space tiles (by i-block) and the bonded terms.  The two halves of the force
    // field thus overlap on different GPUs, there is no charge-grid collective, and one int64 all-reduce of the force buffer
    // per step joins them.  (With PME and world > 1 only; otherwise every rank takes a share of everything.)
    const bool split = role_split(c);
    const int pmeRank = c->world - 1;
    NbDev nbSave = c->nb;
    if (split) {
        if (c->rank == pmeRank) direct = false; else recip = false;
        c->nb = role_nb(c);
    }
    struct Restore { b200md_ctx* c; NbDev saved; ~Restore() { c->nb = saved; } } restore{c, nbSave};
    // Reciprocal space (spread -> FFT/convolution -> gather, in USER atom order: independent of the neighbour list) and
    // direct space (list check / rebuild, tile kernel, bonded terms) are independent until the integrator: fork them onto
    // two streams (also inside the captured step graph).  Both accumulate into the same fixed-point force buffer, so the
    // overlap cannot change the result.  Single-GPU only: with NCCL the collectives of one communicator stay on one stream.
    const bool p2p = c->p2p;
    const bool fork = direct && recip && c->overlapPme && !(c->world > 1 && c->comm && !p2p);
    cudaStream_t sp = fork ? c->streamPme : s;
    if (p2p && !direct) { launch_pos_wait(c->nb, c->cd, s); launches++; }       // nobody else on this stream waits for the owners' position stores
    // The brick path of the spread walks the current list's sorted order, so when it runs beside direct space the
    // fork comes after the list build: the list then cannot flip under it (a rebuild flips at the end of k_build_tiles).
    // On one stream it runs before the build and reads the current list, which is complete even when stale.
    const PmeDev pme = pme_for_launch(c);
    const bool forkAfterList = fork && direct && pme.brickAtoms > 0;
    auto launch_recip = [&]() {
        if (fork) {
            CUDA_CHECK(cudaEventRecord(c->evFork, s));
            CUDA_CHECK(cudaStreamWaitEvent(sp, c->evFork, 0));
        }
        if (recip) {
            launch_pme_spread(c->nb, pme, c->cd, sp, !forkAfterList); launches++;
            if (p2p) { launch_grid_push(c->pme, c->cd, sp); launches++; }
            else if (c->world > 1 && c->comm && !split) {
                int rc = g_nccl.AllReduce(c->gridFixed.p, c->gridFixed.p, (size_t) c->pme.nx*c->pme.ny*c->pme.nz, NCCL_INT64, NCCL_SUM, c->comm, sp);
                if (rc != 0) throw std::runtime_error("ncclAllReduce(grid) failed");
            }
            launch_pme_fft_conv(c->nb, c->pme, c->cd, energy && (split || p2p || c->rank == 0), fft_beside_tiles(c), sp); launches += pme_fft_launch_count(c->pme);
            launch_pme_gather(c->nb, pme, c->cd, sp); launches++;
        }
        if (fork) CUDA_CHECK(cudaEventRecord(c->evJoin, sp));
    };
    if (!forkAfterList) launch_recip();
    // When the chain forks after the list build, the charge grid is zeroed at the head of the step on the chain's stream,
    // beside the list check and build: it needs nothing from them, and as the spread's first node it sat on the chain, which
    // is the step's longest path (DHFR: memset 1.6 us plus a node gap before the spread).
    if (forkAfterList && recip) {
        CUDA_CHECK(cudaEventRecord(c->evForkGrid, s));
        CUDA_CHECK(cudaStreamWaitEvent(sp, c->evForkGrid, 0));
        CUDA_CHECK(cudaMemsetAsync(pme.gridFixed, 0, sizeof(long long)*(size_t) pme.nx*pme.ny*pme.nz, sp));
    }
    if (direct) {
        launch_check_displacement(c->nb, c->cd, s); launches++;
        launch_list_build(c->nb, s); launches += LIST_BUILD_LAUNCHES;
    }
    int bterms = terms & (B200MD_TERM_BONDS | B200MD_TERM_ANGLES | B200MD_TERM_TORSIONS | B200MD_TERM_RB_TORSIONS | B200MD_TERM_CMAP |
                          B200MD_TERM_CUSTOM_TORSIONS);
    if (c->haveNb) bterms |= terms & B200MD_TERM_NB_DIRECT;
    const int nbonded = c->bd.nbonds + c->bd.nangles + c->bd.ntorsions + c->bd.nrb + c->bd.ncmap + c->bd.nexc;
    // the k_bonded branch is counted as one launch whenever it is taken (even when the selected classes have no terms and
    // launch_bonded skips the kernel); k_custom_torsion is counted when it runs
    const bool classic = (bterms & ~B200MD_TERM_CUSTOM_TORSIONS) && nbonded > 0;
    const bool custom = (bterms & B200MD_TERM_CUSTOM_TORSIONS) && c->ctd.nslots > 0;
    const bool bonded = (classic || custom) && !(split && c->rank == pmeRank);
    auto launch_bonded_terms = [&](cudaStream_t sb) {
        BondedDev bd = c->bd; bd.groupMask = groupMask;
        CustomTorsionDev ct = c->ctd; ct.groupMask = groupMask;
        launch_bonded(c->nb, bd, ct, bterms, energy, sb);
        launches += (classic ? 1 : 0) + (custom ? 1 : 0);
    };
    // The bonded terms need nothing from the tile kernel either: on one GPU they fork with the spread onto a stream of their
    // own (not before the list build, whose wrap phase moves molecules in posq) and join before the integrator.
    const bool forkBonded = forkAfterList && bonded;
    if (forkAfterList) launch_recip();
    if (forkBonded) {
        CUDA_CHECK(cudaStreamWaitEvent(c->streamBonded, c->evFork, 0));
        launch_bonded_terms(c->streamBonded);
        CUDA_CHECK(cudaEventRecord(c->evJoinBonded, c->streamBonded));
    }
    if (direct) { launch_pair(c->nb, energy, s); launches += PAIR_LAUNCHES; }
    if (bonded && !forkBonded) launch_bonded_terms(s);
    // p2p: partial forces of the atoms this rank does not own -> the owners' inboxes.  Reciprocal space only ever touches the
    // atoms this rank OWNS (k_pme_gather), so when it runs on its own stream the push does not have to wait for it: it goes
    // out right behind the tile kernel and the bonded terms, beside the FFT chain.
    const bool pushEarly = p2p && fork;
    if (pushEarly) { launch_force_push(c->nb, c->cd, s); launches++; }
    if (fork) CUDA_CHECK(cudaStreamWaitEvent(s, c->evJoin, 0));
    if (forkBonded) CUDA_CHECK(cudaStreamWaitEvent(s, c->evJoinBonded, 0));
    if (p2p) {
        if (!pushEarly) { launch_force_push(c->nb, c->cd, s); launches++; }
        // in the step path k_integrate totals own partial + inboxes; here (energies, getState) the owners total and broadcast
        // so that every rank ends up with every force
        if (!inStep) { launch_force_total(c->nb, c->cd, s); launches += 2; }
    }
    if (c->world > 1 && c->comm) {
        int rc = 0;
        if (!p2p) rc = g_nccl.AllReduce(c->force.p, c->force.p, (size_t) 3*c->npad, NCCL_INT64, NCCL_SUM, c->comm, s);
        if (rc != 0) throw std::runtime_error("ncclAllReduce(force) failed");
        if (energy) {
            rc = g_nccl.AllReduce(c->energy.p, c->energy.p, B200MD_NUM_ENERGY, NCCL_FLOAT64, NCCL_SUM, c->comm, s);
            if (rc != 0) throw std::runtime_error("ncclAllReduce(energy) failed");
        }
    }
    CUDA_CHECK(cudaGetLastError());
    return launches;
}

// The device flags (NbDev::counters) and, if read, the lists' counters, once the stream has finished its work.
struct DevFlags {
    int ct[16], lc[2*LC_STRIDE];
    const int* cur() const { return lc + LC_STRIDE*(ct[CT_CUR] & 1); }       // the current list's counters
};
static DevFlags read_flags(b200md_ctx* c, bool lists) {
    DevFlags f;
    CUDA_CHECK(cudaMemcpyAsync(f.ct, c->counters.p, sizeof(f.ct), cudaMemcpyDeviceToHost, c->stream));
    if (lists) CUDA_CHECK(cudaMemcpyAsync(f.lc, c->listCounters.p, sizeof(f.lc), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    return f;
}
// CT_OVERFLOW codes 2 and 3: a device-side wait gave up
static void raise_timeouts(const DevFlags& f) {
    if (f.ct[CT_OVERFLOW] == 2) throw std::runtime_error("B200 platform: neighbour-list construction timed out at a grid barrier (k_list_prep)");
    if (f.ct[CT_OVERFLOW] == 3) throw std::runtime_error("B200 platform: multi-GPU exchange timed out waiting for a peer rank (every rank must issue the same sequence of calls)");
}

// Sticky device flags are read at EVERY point where the host synchronises with the stream anyway (energy reads, state
// reads, b200md_synchronize), so a problem inside a run of b200md_step calls surfaces at the next state read instead of
// silently dropping pair interactions.
static void check_flags(b200md_ctx* c) {
    if (!c->finalized) return;
    const DevFlags f = read_flags(c, false);
    raise_timeouts(f);
    if (f.ct[CT_OVERFLOW]) throw std::runtime_error("B200 platform: neighbour-list tile capacity exceeded (" + std::to_string(c->nb.maxTiles) + " tiles) during the preceding steps; the trajectory since the last state read is invalid");
}

// After the state was changed from outside (positions, box, parameters, checkpoint): build the list now, synchronously,
// and size the tile pools from what the build actually used.  The step graphs trust the current list and never grow it.
static void prepare_list(b200md_ctx* c) {
    if (!c->listDirty || !c->haveNb) { c->listDirty = false; return; }
    if (c->pmeOnly || (role_split(c) && c->rank == c->world - 1)) { c->listDirty = false; return; }    // keeps no list
    for (int attempt = 0; attempt < 8; attempt++) {
        const NbDev nb = role_nb(c);
        launch_check_displacement(nb, c->cd, c->stream);
        launch_list_build(nb, c->stream);
        c->kernelLaunches += 1 + LIST_BUILD_LAUNCHES;
        const DevFlags f = read_flags(c, true);
        raise_timeouts(f);
        int worst = 0;
        for (int r = 0; r < TILE_REGIONS; r++) worst = std::max(worst, f.cur()[LC_TILES + r]);
        const int cap = c->nb.maxTiles/TILE_REGIONS;
        const bool overflow = f.ct[CT_OVERFLOW] != 0;
        if (!overflow && worst <= (int) (0.8*cap)) { c->listDirty = false; c->listBuilt = true; return; }
        // grow: the counters keep counting past the capacity (flush_tile), so `worst` is the demand even after an overflow
        const int want = std::min(worst_pool_capacity(c), std::max(2*cap, (int) (1.5*worst) + 64));
        if (want <= cap) {
            if (overflow) throw std::runtime_error("B200 platform: neighbour-list tile capacity exceeded and cannot grow (" + std::to_string(c->nb.maxTiles) + " tiles)");
            c->listDirty = false; c->listBuilt = true; return;
        }
        alloc_tile_pools(c, want);
        set_counter(c, CT_OVERFLOW, 0); set_counter(c, CT_REBUILD, 1);
        invalidate_graph(c);
    }
    throw std::runtime_error("B200 platform: neighbour-list tile pools did not converge");
}

extern "C" int b200md_compute(b200md_ctx* ctx, int terms, int want_forces, double* energy) {
    return b200md_compute_groups(ctx, terms, 0xffffffffu, want_forces, energy);
}

extern "C" int b200md_compute_groups(b200md_ctx* ctx, int terms, unsigned int bonded_group_mask, int want_forces, double* energy) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    (void) want_forces;
    require(ctx->finalized, "compute before finalize");
    const bool wantE = energy != nullptr;
    prepare_list(ctx);
    ctx->kernelLaunches += enqueue_forces(ctx, terms, wantE, false, false, bonded_group_mask);
    ctx->forceEvals++;
    if (wantE) {
        double h[B200MD_NUM_ENERGY];
        CUDA_CHECK(cudaMemcpyAsync(h, ctx->energy.p, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
        check_flags(ctx);
        double e = 0;
        if (terms & B200MD_TERM_BONDS) e += h[EN_BOND];
        if (terms & B200MD_TERM_ANGLES) e += h[EN_ANGLE];
        if (terms & B200MD_TERM_TORSIONS) e += h[EN_TORSION];
        if (terms & B200MD_TERM_RB_TORSIONS) e += h[EN_RBTORSION];
        if (terms & B200MD_TERM_CMAP) e += h[EN_CMAP];
        if (terms & B200MD_TERM_CUSTOM_TORSIONS) e += h[EN_CUSTOM_TORSION];
        if (ctx->haveNb) {
            if (terms & B200MD_TERM_NB_DIRECT) {
                e += h[EN_NB] + h[EN_EXC];
                const int m = ctx->nb.method;
                if (m == B200MD_NB_CUTOFF_PERIODIC || m == B200MD_NB_PME)      // ReferenceKernels.cpp:1008-1011
                    e += ctx->dispersionCoefficient/ctx->nb.box.volume;
            }
            if ((terms & B200MD_TERM_NB_RECIP) && ctx->nb.method == B200MD_NB_PME) e += h[EN_RECIP] + ctx->selfEnergy;
        }
        *energy = e;
    }
    API_END(ctx)
}

// ---------------------------------------------------------------- integration
extern "C" int b200md_set_integrator(b200md_ctx* ctx, int kind, double dt, double temperature, double friction, int seed, double tol) {
    API_BEGIN(ctx)
    require(kind >= 0 && kind <= 2, "unknown integrator kind");
    IntegDev& in = ctx->integ;
    in.kind = kind; in.dt = (float) dt; in.tol = (float) tol; in.seed = (unsigned int) seed;
    const double kT = B200MD_BOLTZ*temperature;
    in.kT = (float) kT;
    const double vscale = std::exp(-dt*friction);
    in.vscale = (float) vscale;
    in.fscale = (float) (friction == 0 ? dt : (1-vscale)/friction);
    in.noisescale = (float) (kind == B200MD_INT_LANGEVIN_MIDDLE ? std::sqrt(1-vscale*vscale) : std::sqrt(kT*(1-vscale*vscale)));
    in.dtD = dt; in.tolD = tol; in.kTD = kT; in.vscaleD = vscale;
    in.fscaleD = friction == 0 ? dt : (1-vscale)/friction;
    in.noisescaleD = kind == B200MD_INT_LANGEVIN_MIDDLE ? std::sqrt(1-vscale*vscale) : std::sqrt(kT*(1-vscale*vscale));
    in.stepCounter = ctx->stepCounter.p;
    in.fused = 0; in.cmEveryStep = 0; in.cmScratch = ctx->cmScratch.p; in.blocksDone = ctx->blocksDone.p;
    ctx->dt = dt; ctx->temperature = temperature; ctx->friction = friction;
    ctx->haveIntegrator = true;
    invalidate_graph(ctx);
    API_END(ctx)
}

static int enqueue_step(b200md_ctx* c) {
    // the fused step: the integrate kernel also removes the centre-of-mass motion (frequency 1), zeroes the force buffer
    // for the next step and advances the step counter, so a step is: [check] [rebuild?] pair bonded || spread fft gather ; integrate
    int launches = enqueue_forces(c, B200MD_TERM_ALL, false, true, true);
    IntegDev in = c->integ;
    in.fused = 1;
    in.cmEveryStep = (c->cmFreq == 1) ? 1 : 0;
    in.cmScratch = c->cmScratch.p;
    in.blocksDone = c->blocksDone.p;
    if (c->ccma.ncomp > 0) { launch_ccma_step(c->nb, c->ccma, in, c->stream); launches += 1; }      // before k_integrate: its last block advances the step counter
    launch_integrate(c->nb, c->units, in, c->cd, c->stream); launches += 1;
    return launches;
}

extern "C" int b200md_integrate_only(b200md_ctx* ctx) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    require(ctx->finalized && ctx->haveIntegrator, "integrate before finalize / set_integrator");
    if (ctx->ccma.ncomp > 0) launch_ccma_step(ctx->nb, ctx->ccma, ctx->integ, ctx->stream);
    launch_integrate(ctx->nb, ctx->units, ctx->integ, ctx->cd, ctx->stream);
    ctx->kernelLaunches += 2;
    ctx->velStale = ctx->p2p;
    ctx->time += ctx->dt; ctx->stepCount++;
    CUDA_CHECK(cudaGetLastError());
    API_END(ctx)
}

// Capture `nsteps` steps into *exec.  An executable graph that exists already is updated in place with cudaGraphExecUpdate (a
// box change or a grown tile pool changes kernel parameters, not the topology) and instantiated anew only when the driver
// refuses the update.
static void capture_steps(b200md_ctx* c, int nsteps, cudaGraphExec_t* exec, int* launches) {
    cudaGraph_t g;
    CUDA_CHECK(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    int l = 0;
    try { for (int k = 0; k < nsteps; k++) l += enqueue_step(c); } catch (...) { cudaStreamEndCapture(c->stream, &g); throw; }
    CUDA_CHECK(cudaStreamEndCapture(c->stream, &g));
    *launches = l;
    if (*exec) {
        cudaGraphExecUpdateResultInfo info;
        if (cudaGraphExecUpdate(*exec, g, &info) == cudaSuccess) { cudaGraphDestroy(g); return; }
        (void) cudaGetLastError();          // the refusal is not sticky: fall back to a new instantiation
    }
    if (*exec) { cudaGraphExecDestroy(*exec); *exec = nullptr; }
    // One GPU: the graph runs each kernel node at its own priority (launch_high), not at the priority of c->stream, so the
    // reciprocal-space chain and the bonded terms take the SM slots that the tile kernel's CTAs hand back.  An update in
    // place keeps the priorities: every capture gives the same nodes the same ones.
    const cudaError_t e = cudaGraphInstantiate(exec, g, c->world == 1 ? cudaGraphInstantiateFlagUseNodePriority : 0);
    cudaGraphDestroy(g);
    CUDA_CHECK(e);
    c->graphInstantiations++;
}

extern "C" int b200md_step(b200md_ctx* ctx, int nsteps) {
    API_BEGIN(ctx)
    require(ctx->finalized && ctx->haveIntegrator, "step before finalize / set_integrator");
    b200md_ctx* c = ctx;
    int remaining = nsteps;
    prepare_list(c);      // the state was changed from outside: the step graphs trust the current list
    if (!c->stepStateValid) {
        CUDA_CHECK(cudaMemsetAsync(c->force.p, 0, sizeof(long long)*3*c->npad, c->stream));
        if (c->cmFreq == 1) {
            IntegDev in = c->integ;
            in.cmScratch = c->cmScratch.p;
            sync_velocities(c);
            launch_cm_prime(c->nb, in, c->cd, c->stream);
        }
        c->stepStateValid = true;
    }
    while (remaining > 0) {
        if (c->cmFreq > 1 && c->stepCount % c->cmFreq == 0) { sync_velocities(c); launch_remove_cm(c->nb, c->cmScratch.p, c->stream); c->kernelLaunches += 2; }
        int done = 1;
        if (c->useGraph) {
            // the multi-step graph may not straddle a centre-of-mass removal that lives outside the graph; it is captured only
            // when this call can use it (the plugin only ever steps one at a time)
            int untilCm = (c->cmFreq > 1) ? (int) (c->cmFreq - c->stepCount % c->cmFreq) : remaining;
            if (c->graphSteps > 1 && remaining >= c->graphSteps && untilCm >= c->graphSteps) {
                if (!c->multiValid) { int l; capture_steps(c, c->graphSteps, &c->multiGraph, &l); c->stepLaunches = l/c->graphSteps; c->multiValid = true; }
                CUDA_CHECK(cudaGraphLaunch(c->multiGraph, c->stream));
                done = c->graphSteps;
            }
            else {
                if (!c->graphValid) { capture_steps(c, 1, &c->stepGraph, &c->stepLaunches); c->graphValid = true; }
                CUDA_CHECK(cudaGraphLaunch(c->stepGraph, c->stream));
            }
            c->kernelLaunches += (int64_t) c->stepLaunches*done;
        }
        else
            c->kernelLaunches += enqueue_step(c);
        c->velStale = c->p2p;
        c->forceEvals += done;
        c->stepCount += done;
        c->time += c->dt*done;
        remaining -= done;
    }
    CUDA_CHECK(cudaGetLastError());
    API_END(ctx)
}

extern "C" int b200md_kinetic_energy(b200md_ctx* ctx, double* ke) {
    API_BEGIN(ctx)
    require(ctx->finalized, "kinetic_energy before finalize");
    const bool shifted = ctx->haveIntegrator && ctx->integ.kind != B200MD_INT_LANGEVIN_MIDDLE;
    const double shift = !shifted ? 0.0 : ctx->mixed() ? 0.5*ctx->integ.dtD : (double) (0.5f*ctx->integ.dt);
    sync_positions(ctx); sync_velocities(ctx);
    CUDA_CHECK(cudaMemsetAsync(ctx->energy.p + EN_KE, 0, sizeof(double), ctx->stream));
    launch_kinetic_energy(ctx->nb, ctx->units, ctx->integ, shift, ctx->stream);
    launch_ccma_kinetic(ctx->nb, ctx->ccma, shift, 1e-4f, ctx->stream);
    ctx->kernelLaunches++;
    CUDA_CHECK(cudaMemcpyAsync(ke, ctx->energy.p + EN_KE, sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    check_flags(ctx);
    API_END(ctx)
}
extern "C" int b200md_apply_constraints(b200md_ctx* ctx, double tol) {
    API_BEGIN(ctx)
    sync_positions(ctx);
    launch_constrain_positions(ctx->nb, ctx->units, tol, ctx->stream);
    launch_ccma_apply(ctx->nb, ctx->ccma, false, tol, ctx->stream);
    ctx->kernelLaunches++;
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    API_END(ctx)
}
extern "C" int b200md_apply_velocity_constraints(b200md_ctx* ctx, double tol) {
    API_BEGIN(ctx)
    ctx->stepStateValid = false;
    sync_positions(ctx); sync_velocities(ctx);
    launch_constrain_velocities(ctx->nb, ctx->units, tol, ctx->stream);
    launch_ccma_apply(ctx->nb, ctx->ccma, true, tol, ctx->stream);
    ctx->kernelLaunches++;
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    API_END(ctx)
}

// ---------------------------------------------------------------- multi-GPU
extern "C" int b200md_comm_unique_id(void* id128) {
    std::string err;
    if (!g_nccl.load(err)) { g_create_error = err; return -1; }
    return g_nccl.GetUniqueId(id128) == 0 ? 0 : -1;
}
extern "C" int b200md_comm_init(b200md_ctx* ctx, int rank, int world, const void* id128) {
    API_BEGIN(ctx)
    require(!ctx->finalized, "comm_init must precede finalize");
    require(!ctx->mixed() || world <= 1, "comm_init: mixed precision is not supported in multi-GPU runs (use Precision=single)");
    std::string err;
    if (!g_nccl.load(err)) throw std::runtime_error(err);
    NcclApi::Uid uid; memcpy(uid.b, id128, 128);
    int rc = g_nccl.CommInitRank(&ctx->comm, world, uid, rank);
    if (rc != 0) throw std::runtime_error(std::string("ncclCommInitRank failed: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(rc) : "?"));
    ctx->rank = rank; ctx->world = world;
    // one eager collective: NCCL sets its transports up lazily on the first call, which must not happen inside a
    // CUDA-graph capture (the step graph contains the force all-reduce)
    DevBuf<long long> warm; warm.alloc(64); warm.zero();
    rc = g_nccl.AllReduce(warm.p, warm.p, 64, NCCL_INT64, NCCL_SUM, ctx->comm, ctx->stream);
    if (rc != 0) throw std::runtime_error("ncclAllReduce warm-up failed");
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    API_END(ctx)
}

// ---------------------------------------------------------------- stand-alone reciprocal space (CalcPmeReciprocalForceKernel)
extern "C" int b200md_pme_create(b200md_ctx** out, int device, int natoms, int nx, int ny, int nz, double alpha) {
    int rc = b200md_create(out, device, natoms);
    if (rc != 0) return rc;
    b200md_ctx* c = *out;
    c->pmeOnly = true;
    std::vector<double> one(natoms, 1.0), zero(natoms, 0.0);
    b200md_nonbonded_desc d = b200md_nonbonded_desc{};
    d.method = B200MD_NB_PME; d.cutoff = 0.01; d.ewald_alpha = alpha; d.grid[0] = nx; d.grid[1] = ny; d.grid[2] = nz;
    rc = b200md_set_masses(c, one.data());
    if (rc == 0) rc = b200md_set_nonbonded(c, &d, zero.data(), one.data(), zero.data());
    return rc;          // finalised at the first exec, when the box is known
}

extern "C" int b200md_pme_exec(b200md_ctx* ctx, const float* posq, const double box[9], int include_energy, float* force4, double* energy) {
    if (!ctx) return -1;
    if (!ctx->finalized || std::memcmp(box, ctx->boxA, 3*sizeof(double)) || std::memcmp(box+3, ctx->boxB, 3*sizeof(double)) || std::memcmp(box+6, ctx->boxC, 3*sizeof(double))) {
        int rc = b200md_set_box(ctx, box, box+3, box+6);
        if (rc == 0 && !ctx->finalized) rc = b200md_finalize(ctx);
        if (rc != 0) return rc;
    }
    API_BEGIN(ctx)
    require(ctx->pmeOnly, "b200md_pme_exec on a context that was not made by b200md_pme_create");
    b200md_ctx* c = ctx;
    const float sk = (float) std::sqrt(B200MD_ONE_4PI_EPS0);
    std::vector<float4> h(c->npad, make_float4(0, 0, 0, 0));
    for (int i = 0; i < c->natoms; i++) h[i] = make_float4(posq[4*i], posq[4*i+1], posq[4*i+2], posq[4*i+3]*sk);
    CUDA_CHECK(cudaMemcpyAsync(c->posq.p, h.data(), sizeof(float4)*c->npad, cudaMemcpyHostToDevice, c->stream));
    c->kernelLaunches += enqueue_forces(c, B200MD_TERM_NB_RECIP, include_energy != 0);
    c->forceEvals++;
    c->hforce.resize((size_t) 3*c->npad);
    double he[B200MD_NUM_ENERGY] = {0};
    CUDA_CHECK(cudaMemcpyAsync(c->hforce.data(), c->force.p, sizeof(long long)*3*c->npad, cudaMemcpyDeviceToHost, c->stream));
    if (include_energy) CUDA_CHECK(cudaMemcpyAsync(he, c->energy.p, sizeof(he), cudaMemcpyDeviceToHost, c->stream));
    CUDA_CHECK(cudaStreamSynchronize(c->stream));
    const double s = 1.0/B200MD_FORCE_SCALE;
    for (int i = 0; i < c->natoms; i++)
        for (int k = 0; k < 3; k++) force4[4*i+k] = (float) (s*(double) c->hforce[(size_t) k*c->npad + i]);
    if (energy) *energy = include_energy ? he[EN_RECIP] : 0.0;
    API_END(ctx)
}

// ---------------------------------------------------------------- introspection
extern "C" int b200md_get_stats(b200md_ctx* ctx, b200md_stats* out) {
    API_BEGIN(ctx)
    memset(out, 0, sizeof(*out));
    out->natoms = ctx->natoms; out->padded_atoms = ctx->npad; out->num_blocks = ctx->nblocks;
    if (ctx->finalized) {
        launch_count_pairs(ctx->nb, ctx->stream);
        const DevFlags f = read_flags(ctx, true);
        int masks = 0;
        for (int r = 0; r < TILE_REGIONS; r++) masks += f.cur()[LC_MASKS + r];
        out->num_tiles = f.cur()[LC_USED]; out->num_mask_tiles = masks; out->overflow = f.ct[CT_OVERFLOW]; out->list_builds = f.ct[CT_BUILDS]; out->pairs_in_cutoff = f.ct[CT_PAIRS];
    }
    out->force_evals = ctx->forceEvals; out->kernel_launches = ctx->kernelLaunches; out->graph_instantiations = ctx->graphInstantiations;
    out->pme_grid[0] = ctx->pme.nx; out->pme_grid[1] = ctx->pme.ny; out->pme_grid[2] = ctx->pme.nz; out->ewald_alpha = ctx->pme.alpha;
    API_END(ctx)
}

extern "C" int b200md_time_phase(b200md_ctx* ctx, int phase, int reps, double* ms_mean) {
    API_BEGIN(ctx)
    require(ctx->finalized, "time_phase before finalize");
    b200md_ctx* c = ctx;
    prepare_list(c);
    c->stepStateValid = false;            // phases 0, 3, 6 accumulate into the force buffer, phase 5 flips the list
    cudaStream_t s = c->stream;
    const NbDev nbv = role_nb(c);        // the sharding the step graphs use
    CommDev local{}; local.world = 1;   // phases are timed rank-locally (no peer traffic, no waits)
    cudaEvent_t e0, e1;
    CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
    double total = 0;
    // the integrate phase mutates the state: positions and velocities are restored before every repetition, the step
    // counter (which each repetition advances, as a step does) once at the end
    Snapshot state, counter;
    require(phase != 7 || c->ctd.nslots > 0, "time_phase(custom torsions): the System has none");
    if (phase == 4) {
        require(c->haveIntegrator, "time_phase(integrate) before set_integrator");
        state.parts = state_spans(c, ST_POS | ST_VEL); state.save(s);
        counter.parts = {{c->stepCounter.p, sizeof(unsigned long long)}}; counter.save(s);
    }
    for (int r = -2; r < reps; r++) {
        if (phase == 4) state.restore(s);
        if (phase == 5) set_counter(c, CT_REBUILD, 1);     // the list is not marked dirty: the next step adds no synchronous rebuild
        if (phase == 0) { CUDA_CHECK(cudaMemsetAsync(&c->counters.p[CT_CURSOR], 0, sizeof(int), s)); CUDA_CHECK(cudaMemsetAsync(&c->counters.p[CT_PAIRSTART], 0, sizeof(int), s)); }      // the SM-partitioned tile kernel's cursor starts from tile 0
        CUDA_CHECK(cudaEventRecord(e0, s));
        switch (phase) {
            case 0: launch_pair(nbv, false, s); break;
            case 1: launch_pme_spread(nbv, pme_for_launch(c), local, s); break;
            case 2: launch_pme_fft_conv(nbv, c->pme, local, false, fft_beside_tiles(c), s); break;
            case 3: launch_pme_gather(nbv, pme_for_launch(c), local, s); break;
            case 4: launch_integrate(nbv, c->units, c->integ, local, s); break;
            case 5: launch_list_build(nbv, s); break;
            case 6: launch_bonded(nbv, c->bd, c->ctd, B200MD_TERM_ALL, false, s); break;
            case 7: launch_custom_torsion(nbv, c->ctd, false, s); break;
            default: throw std::runtime_error("unknown phase");
        }
        CUDA_CHECK(cudaEventRecord(e1, s));
        CUDA_CHECK(cudaEventSynchronize(e1));
        float ms = 0; CUDA_CHECK(cudaEventElapsedTime(&ms, e0, e1));
        if (r >= 0) total += ms;
    }
    if (phase == 4) {
        state.restore(s); counter.restore(s);
        CUDA_CHECK(cudaStreamSynchronize(s));
    }
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    *ms_mean = total/std::max(1, reps);
    API_END(ctx)
}

// stand-alone FFT for parity tests of the bespoke transform
static int fft_standalone(int device, int nx, int ny, int nz, const float* in, float* out, bool forward) {
    try {
        CUDA_CHECK(cudaSetDevice(device));
        PmeDev p{}; p.nx = nx; p.ny = ny; p.nz = nz; p.nzc = nz/2 + 1;
        DevBuf<real> grid; DevBuf<real2> cg; DevBuf<real2> tw[3];
        grid.alloc((size_t) nx*ny*nz); cg.alloc((size_t) nx*ny*p.nzc);
        p.grid = grid.p; p.cgrid = cg.p;
        const int n[3] = {nx, ny, nz};
        for (int d = 0; d < 3; d++) make_fft_plan(n[d], p.plan[d], tw[d]);
        int maxSmem = 0;
        cudaDeviceGetAttribute(&maxSmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
        require(fft_plane_smem_bytes(ny, nz) <= (size_t) maxSmem && fft_line_smem_bytes(nx) <= (size_t) maxSmem, "grid too large for shared memory");
        // host API is fp32 (TestCudaFFT3D-style checks); the device transform is double
        if (forward) {
            std::vector<real> h(grid.n);
            for (size_t i = 0; i < grid.n; i++) h[i] = (real) in[i];
            CUDA_CHECK(cudaMemcpy(grid.p, h.data(), sizeof(real)*grid.n, cudaMemcpyHostToDevice));
            launch_fft3d_r2c(p, 0);
            CUDA_CHECK(cudaDeviceSynchronize());
            std::vector<real> o(2*cg.n);
            CUDA_CHECK(cudaMemcpy(o.data(), cg.p, sizeof(real2)*cg.n, cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < 2*cg.n; i++) out[i] = (float) o[i];
        }
        else {
            std::vector<real> h(2*cg.n);
            for (size_t i = 0; i < 2*cg.n; i++) h[i] = (real) in[i];
            CUDA_CHECK(cudaMemcpy(cg.p, h.data(), sizeof(real2)*cg.n, cudaMemcpyHostToDevice));
            launch_fft3d_c2r(p, 0);
            CUDA_CHECK(cudaDeviceSynchronize());
            std::vector<real> o(grid.n);
            CUDA_CHECK(cudaMemcpy(o.data(), grid.p, sizeof(real)*grid.n, cudaMemcpyDeviceToHost));
            for (size_t i = 0; i < grid.n; i++) out[i] = (float) o[i];
        }
        return 0;
    } catch (std::exception& e) { g_create_error = e.what(); return -1; }
}
extern "C" int b200md_fft3d_r2c(int device, int nx, int ny, int nz, const float* in, float* out) { return fft_standalone(device, nx, ny, nz, in, out, true); }
extern "C" int b200md_fft3d_c2r(int device, int nx, int ny, int nz, const float* in, float* out) { return fft_standalone(device, nx, ny, nz, in, out, false); }
