// engine.cu -- host side of libb200md.so: the C-ABI of include/b200md.h over the CUDA kernels of this directory.
// No CPU fallback exists: every compute entry point needs a CUDA device and fails loudly without one.
#include "engine.h"
#include "custom_interp.h"
#include "rmsd.h"
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
// One class of custom terms (B200MD_CUSTOM_*), in the caller's order: per term its expression, its atoms at the class's
// width (CUSTOM_NAMES: a torsion's four, a bond's two, an external's one, an angle's three, a compound bond's eight with the
// unused ones -1), params [n][stride] and group; per expression its first program (exprProg[nexpr]: the number of programs,
// 1 + the class's number of variables per expression, 1 + 3 particles for a compound bond), its particles per term and
// whether its point functions take the minimum image (both 0 but for compound bonds); the programs (op, arg, imm,
// progStart).  slot[i] is the slot of term i in its kernel's layout.
struct CustomClass {
    int n = 0, stride = 0, nexpr = 0;
    std::vector<int> atoms, expr, exprProg, nparticles, periodic, progStart, op, arg, slot;
    std::vector<double> imm, params; std::vector<unsigned char> group;
};
// The classes [first, last) one kernel runs, in its layout (finalize, layout_custom): k_custom the torsions, bonds, externals
// and angles (CustomDev), k_compound the compound bonds (CompoundDev), its centroid instantiation the centroid bonds (a second
// CompoundDev).
struct CustomSlots {
    int first, last;
    int nslots = 0, stride = 0;
    DevBuf<int> atomsDev, exprDev, exprClassDev, exprParticlesDev, exprPeriodicDev, exprProgDev, progStartDev;
    DevBuf<int2> codeDev; DevBuf<double> immDev, paramsDev; DevBuf<unsigned char> groupDev;
};
// The groups of the centroid bonds (CentroidDev): CSR over atoms with their normalised weights, as the set call got them; on the
// device besides the centres, the derivatives per slot and the scatter entries (finalize, upload_custom)
struct CentroidGroups {
    std::vector<int> start, atoms; std::vector<double> weight;
    DevBuf<int> startDev, atomsDev; DevBuf<double> weightDev, centerDev, derivDev, scatterWeightDev; DevBuf<int4> scatterDev;
};
enum { CUSTOM_CLASSES = 6 };
// Every custom class and the global values (one slot space for all classes)
struct CustomTable {
    CustomClass cls[CUSTOM_CLASSES];
    CustomSlots kernel[3] = {{B200MD_CUSTOM_TORSION, B200MD_CUSTOM_COMPOUND}, {B200MD_CUSTOM_COMPOUND, B200MD_CUSTOM_COMPOUND + 1},
                             {B200MD_CUSTOM_CENTROID, B200MD_CUSTOM_CENTROID + 1}};
    CentroidGroups groups;
    std::vector<double> globals;
    DevBuf<double> globalsDev;
    CustomSlots& kernel_of(int cls) { return kernel[cls == B200MD_CUSTOM_COMPOUND ? 1 : cls == B200MD_CUSTOM_CENTROID ? 2 : 0]; }
    // the params of the classes of s in its slot layout (padding slots 0)
    std::vector<double> slot_params(const CustomSlots& s) const {
        std::vector<double> p((size_t) s.nslots*s.stride, 0.0);
        for (int k = s.first; k < s.last; k++) {
            const CustomClass& t = cls[k];
            for (int i = 0; i < t.n; i++)
                std::copy(t.params.begin() + (size_t) i*t.stride, t.params.begin() + (size_t) (i+1)*t.stride, p.begin() + (size_t) t.slot[i]*s.stride);
        }
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

// The multi-GPU scheme of a context, decided once by b200md_finalize (MG_SINGLE before it):
//   MG_SINGLE       world == 1
//   MG_P2P          the peer-memory data plane (comm.cu, DESIGN.md section 5): B200MD_MGPU unset or not "nccl"
//   MG_NCCL_SPLIT   B200MD_MGPU=nccl with PME: the last rank does reciprocal space for every atom and nothing else, the others
//                   share the direct-space tiles and the bonded terms; an NCCL all-reduce of the force buffer joins them
//   MG_NCCL_SHARED  B200MD_MGPU=nccl without PME: every rank takes a share of everything, joined the same way
enum MultiGpu { MG_SINGLE, MG_P2P, MG_NCCL_SPLIT, MG_NCCL_SHARED };

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
    CustomTable custom;
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
    CustomDev ctd{};
    CompoundDev cpd{};
    CompoundDev ccd{};          // the centroid bonds' programs and slots
    CentroidDev cen{};
    // generalized Born (b200md_set_gbsa): the force's settings and per-atom parameters as given, their device form and the
    // stream the chain runs on beside the tile kernel (created at finalize when there is one)
    struct {
        bool have = false;
        int method = 0;
        double cutoff = 0, solute = 1, solvent = 78.5, surface = 0;
        std::vector<double> charge, radius, scale;
        DevBuf<float> chargeDev; DevBuf<double2> radiusDev; DevBuf<double> atomRadiusDev, bornR, chain, bornForce;
        DevBuf<long long> bornSum, dEdB;
        cudaStream_t stream = nullptr;
        cudaEvent_t evFork = nullptr, evJoin = nullptr;
    } gbsa;
    GbsaDev gbd{};
    // CustomNonbondedForce objects (b200md_set_custom_nonbonded): the shared method, cutoff and excluded pairs, every object's
    // programs, parameters, switching distance, group and long-range coefficient as given, the tables, their device form and the
    // stream the pair kernel runs on beside the tile kernel (created at finalize when there are objects)
    struct {
        bool have = false;
        int method = 0, nobj = 0, stride = 0;
        double cutoff = 0;
        std::vector<int> progStart, op, arg, nparams, group; std::vector<double> imm, params, switchDist, lrc;
        std::vector<int2> excl;
        std::vector<int4> tableDims; std::vector<int> tableStart; std::vector<double> tableValues;
        DevBuf<int> progStartDev, nparamsDev, groupDev, tableStartDev; DevBuf<int2> codeDev; DevBuf<int4> tableDimsDev;
        DevBuf<double> immDev, paramsDev, switchDev, tableValuesDev;
        cudaStream_t stream = nullptr;
        cudaEvent_t evFork = nullptr, evJoin = nullptr;
    } cnb;
    CnbDev cnd{};
    // RMSDForce objects (b200md_set_rmsd): their particle lists one after the other, the reference position of every entry
    // centred over its object, and the device form
    struct {
        std::vector<int> start, atoms, entryObj; std::vector<double> ref, refSq; std::vector<unsigned char> group;
        DevBuf<int> startDev, atomsDev, entryObjDev; DevBuf<double> refDev, refSqDev, sums, solved; DevBuf<unsigned char> groupDev;
    } rmsd;
    RmsdDev rmd{};
    // CustomCVForce (b200md_set_cv_forces): the number of collective variables, their force snapshots and coefficients; evCv
    // orders this context's stream against another's (state copies and force snapshots)
    struct {
        int n = 0;
        DevBuf<long long> forces; DevBuf<double> coeff; std::vector<double> hcoeff;
    } cv;
    CvDev cvd{};
    cudaEvent_t evCv = nullptr;
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
    MultiGpu mg = MG_SINGLE;
    // peer-memory data plane (comm.cu): one window per rank, mapped by every other rank with CUDA IPC
    CommDev cd{};                        // world == 1 unless MG_P2P
    char* window = nullptr; size_t windowBytes = 0;
    void* peerMapped[B200MD_MAX_RANKS] = {nullptr};
    DevBuf<unsigned long long> commCounters;   // [0] epoch, [1] posNeed
    DevBuf<unsigned int> commDone;             // [CH_COUNT]
    bool velStale = false;               // MG_P2P: the velocities of foreign atoms are behind (only owners integrate)
    std::vector<float4> hbuf4, hcorr4;
    std::vector<int> hoffset;
    std::vector<long long> hforce;
};

#define API_BEGIN(ctx) if (!(ctx)) return -1; try { CUDA_CHECK(cudaSetDevice((ctx)->device));
#define API_END(ctx) } catch (std::exception& e) { (ctx)->err = e.what(); return -1; } return 0;

static void check_flags(b200md_ctx* c);
static void sync_velocities(b200md_ctx* c);
static void sync_positions(b200md_ctx* c);
static void setup_gbsa(b200md_ctx* c);
static void setup_custom_nonbonded(b200md_ctx* c);
static void setup_rmsd(b200md_ctx* c);
static void setup_cv(b200md_ctx* c);
static void host_set_state(b200md_ctx* c);

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
    if (ctx->evCv) cudaEventDestroy(ctx->evCv);
    if (ctx->gbsa.stream) cudaStreamDestroy(ctx->gbsa.stream);
    if (ctx->gbsa.evFork) cudaEventDestroy(ctx->gbsa.evFork);
    if (ctx->gbsa.evJoin) cudaEventDestroy(ctx->gbsa.evJoin);
    if (ctx->cnb.stream) cudaStreamDestroy(ctx->cnb.stream);
    if (ctx->cnb.evFork) cudaEventDestroy(ctx->cnb.evFork);
    if (ctx->cnb.evJoin) cudaEventDestroy(ctx->cnb.evJoin);
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
// What the custom classes differ in on the host: the names in the messages of their calls (what the set call counts: programs,
// or expressions for compound and centroid bonds), the atoms per term (a centroid bond's are groups), whether a term's atoms
// join the molecules that wrap together (not an external's, which acts on one particle, nor a compound bond's, which reads
// continuous coordinates and may tie two molecules that must keep wrapping apart, nor a centroid bond's, whose groups would
// otherwise tie a protein to every water near it), the term bit and the bonded kind.
struct CustomNames {
    const char* call; const char* term; const char* per; const char* unit; const char* update; const char* terms;
    int width; bool joins; int bit; int kind;
};
static const CustomNames CUSTOM_NAMES[CUSTOM_CLASSES] = {
    {"set_custom_torsions", "custom torsion", "torsion", "program", "update_custom_torsion_params", "torsions", 4, true,
     B200MD_TERM_CUSTOM_TORSIONS, B200MD_BONDED_CUSTOM_TORSIONS},
    {"set_custom_bonds", "custom bond", "bond", "program", "update_custom_bond_params", "bonds", 2, true,
     B200MD_TERM_CUSTOM_BONDS, B200MD_BONDED_CUSTOM_BONDS},
    {"set_custom_externals", "custom external", "particle", "program", "update_custom_external_params", "particles", 1, false,
     B200MD_TERM_CUSTOM_EXTERNALS, B200MD_BONDED_CUSTOM_EXTERNALS},
    {"set_custom_angles", "custom angle", "angle", "program", "update_custom_angle_params", "angles", 3, true,
     B200MD_TERM_CUSTOM_ANGLES, B200MD_BONDED_CUSTOM_ANGLES},
    {"set_custom_compound", "custom compound bond", "bond", "expression", "update_custom_compound_params", "bonds", B200MD_CUSTOM_MAX_PARTICLES, false,
     B200MD_TERM_CUSTOM_COMPOUND, B200MD_BONDED_CUSTOM_COMPOUND},
    {"set_custom_centroid", "custom centroid bond", "bond", "expression", "update_custom_centroid_params", "bonds", B200MD_CUSTOM_MAX_PARTICLES, false,
     B200MD_TERM_CUSTOM_CENTROID, B200MD_BONDED_CUSTOM_CENTROID}};
// compound and centroid bonds: expressions of the coordinates of up to 8 particles (atoms or group centres) per term
static bool custom_points(int cls) { return cls == B200MD_CUSTOM_COMPOUND || cls == B200MD_CUSTOM_CENTROID; }

// A program set of class cls (b200md_set_custom_torsions / _bonds / _externals / _angles / _compound / _centroid): nexpr
// expressions, the programs of one after the other's (1 + the class's number of variables each; 1 + 3 nparticles[p] for
// compound and centroid bonds), prog_start well formed and every program passing custom_check_program (nglobals < 0: GLOBAL
// operands are checked at finalize).  Returns the instructions as (opcode, operand) and, in exprProg, every expression's first program and, last,
// the number of programs.
static std::vector<int2> check_programs(int cls, int nexpr, const int* nparticles, const int* prog_start, const int* op, const int* arg,
                                        int stride, int nglobals, std::vector<int>& exprProg) {
    const bool compound = custom_points(cls);
    const std::string call = CUSTOM_NAMES[cls].call;
    require(nexpr >= 0, (call + ": negative number of " + CUSTOM_NAMES[cls].unit + "s").c_str());
    require(stride >= 0 && stride <= B200MD_CUSTOM_MAX_PARAMS, (call + ": more than 16 parameters per " + CUSTOM_NAMES[cls].per).c_str());
    require(nexpr == 0 || prog_start[0] == 0, (call + ": prog_start[0] must be 0").c_str());
    exprProg.assign(nexpr + 1, 0);
    for (int p = 0; p < nexpr; p++) {
        if (compound)
            require(nparticles[p] >= 1 && nparticles[p] <= B200MD_CUSTOM_MAX_PARTICLES,
                    (call + ": an expression must join 1 to 8 " + (cls == B200MD_CUSTOM_CENTROID ? "groups" : "particles")).c_str());
        exprProg[p+1] = exprProg[p] + 1 + (compound ? 3*nparticles[p] : custom_num_vars(cls));
    }
    const int nq = exprProg[nexpr];
    for (int q = 0; q < nq; q++) require(prog_start[q+1] >= prog_start[q], (call + ": prog_start must not decrease").c_str());
    const int total = nexpr ? prog_start[nq] : 0;
    std::vector<int2> code(total);
    for (int k = 0; k < total; k++) code[k] = make_int2(op[k], arg[k]);
    for (int p = 0; p < nexpr; p++)
        for (int q = exprProg[p]; q < exprProg[p+1]; q++) {
            const char* why = custom_check_program(cls, code.data(), prog_start[q], prog_start[q+1], stride, nglobals, compound ? nparticles[p] : 0);
            if (why) throw std::runtime_error(std::string(why) + " (program " + std::to_string(q) + ")");
        }
    return code;
}
// The terms of class cls: term i evaluates expression expr[i] on the atoms atoms[w*i .. w*i+w-1] (w = the class's width; a
// compound bond's unused slots -1; a centroid bond's are groups, indices below nindex).  nparticles and periodic (per
// expression) are read for compound and centroid bonds only.
static void set_custom(b200md_ctx* ctx, int cls, int nexpr, const int* nparticles, const int* periodic, const int* prog_start, const int* op,
                       const int* arg, const double* imm, int stride, int n, const int* expr, const int* atoms, const double* params,
                       int nindex = -1) {
    const CustomNames& nm = CUSTOM_NAMES[cls];
    const bool compound = custom_points(cls), centroid = cls == B200MD_CUSTOM_CENTROID;
    if (nindex < 0) nindex = ctx->natoms;
    check_set(ctx, nm.call, n);
    require(ctx->world == 1, (std::string(nm.term) + "s are not supported in multi-GPU runs").c_str());
    std::vector<int> exprProg;
    check_programs(cls, nexpr, nparticles, prog_start, op, arg, stride, -1, exprProg);
    const int w = nm.width;
    for (int i = 0; i < n; i++) {
        require(expr[i] >= 0 && expr[i] < nexpr, (std::string(nm.term) + ": " + nm.unit + " index out of range").c_str());
        for (int k = 0; k < w; k++) {
            const int a = atoms[w*i + k];
            if (!compound || k < nparticles[expr[i]])
                require(a >= 0 && a < nindex, (std::string(nm.term) + (centroid ? ": group" : ": atom") + " index out of range").c_str());
            else require(a == -1, (std::string(nm.term) + (centroid ? ": an unused group" : ": an unused atom") + " slot must be -1").c_str());
        }
    }
    CustomClass& t = ctx->custom.cls[cls];            // its group stays: groups may come before the terms
    const int nq = exprProg[nexpr];
    t.n = n; t.stride = stride; t.nexpr = nexpr; t.exprProg.swap(exprProg);
    t.nparticles.assign(nexpr, 0); t.periodic.assign(nexpr, 0);
    if (compound) { t.nparticles.assign(nparticles, nparticles + nexpr); t.periodic.assign(periodic, periodic + nexpr); }
    t.progStart.assign(prog_start, prog_start + (nexpr ? nq + 1 : 0));
    const int total = nexpr ? prog_start[nq] : 0;
    t.op.assign(op, op + total); t.arg.assign(arg, arg + total); t.imm.assign(imm, imm + total);
    t.expr.assign(expr, expr + n); t.atoms.assign(atoms, atoms + (size_t) w*n);
    t.params.assign(params, params + (size_t) n*stride);
}
extern "C" int b200md_set_custom_torsions(b200md_ctx* ctx, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                          int stride, int n, const int* prog, const int* atoms, const double* params) {
    API_BEGIN(ctx)
    set_custom(ctx, B200MD_CUSTOM_TORSION, nprog, nullptr, nullptr, prog_start, op, arg, imm, stride, n, prog, atoms, params);
    API_END(ctx)
}
extern "C" int b200md_set_custom_bonds(b200md_ctx* ctx, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                       int stride, int n, const int* prog, const int* atoms, const double* params) {
    API_BEGIN(ctx)
    set_custom(ctx, B200MD_CUSTOM_BOND, nprog, nullptr, nullptr, prog_start, op, arg, imm, stride, n, prog, atoms, params);
    API_END(ctx)
}
extern "C" int b200md_set_custom_externals(b200md_ctx* ctx, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                           int stride, int n, const int* prog, const int* atoms, const double* params) {
    API_BEGIN(ctx)
    set_custom(ctx, B200MD_CUSTOM_EXTERNAL, nprog, nullptr, nullptr, prog_start, op, arg, imm, stride, n, prog, atoms, params);
    API_END(ctx)
}
extern "C" int b200md_set_custom_angles(b200md_ctx* ctx, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                        int stride, int n, const int* prog, const int* atoms, const double* params) {
    API_BEGIN(ctx)
    set_custom(ctx, B200MD_CUSTOM_ANGLE, nprog, nullptr, nullptr, prog_start, op, arg, imm, stride, n, prog, atoms, params);
    API_END(ctx)
}
extern "C" int b200md_set_custom_compound(b200md_ctx* ctx, int nexpr, const int* nparticles, const int* periodic, const int* prog_start,
                                          const int* op, const int* arg, const double* imm, int stride, int n, const int* expr,
                                          const int* atoms, const double* params) {
    API_BEGIN(ctx)
    set_custom(ctx, B200MD_CUSTOM_COMPOUND, nexpr, nparticles, periodic, prog_start, op, arg, imm, stride, n, expr, atoms, params);
    API_END(ctx)
}
extern "C" int b200md_set_custom_centroid(b200md_ctx* ctx, int nexpr, const int* ngroups_per_bond, const int* periodic, const int* prog_start,
                                          const int* op, const int* arg, const double* imm, int stride, int n, const int* expr,
                                          const int* groups, const double* params, int ngroups, const int* group_start,
                                          const int* group_atoms, const double* group_weights) {
    API_BEGIN(ctx)
    check_set(ctx, "set_custom_centroid", ngroups);
    require(ngroups == 0 || group_start[0] == 0, "set_custom_centroid: group_start[0] must be 0");
    for (int g = 0; g < ngroups; g++) require(group_start[g+1] > group_start[g], "custom centroid bond: a group must hold at least one atom");
    const int total = ngroups ? group_start[ngroups] : 0;
    for (int k = 0; k < total; k++) {
        require(group_atoms[k] >= 0 && group_atoms[k] < ctx->natoms, "custom centroid bond: atom index of a group out of range");
        require(std::isfinite(group_weights[k]), "custom centroid bond: a group weight is not finite");
    }
    set_custom(ctx, B200MD_CUSTOM_CENTROID, nexpr, ngroups_per_bond, periodic, prog_start, op, arg, imm, stride, n, expr, groups, params, ngroups);
    CentroidGroups& g = ctx->custom.groups;
    g.start.assign(group_start, group_start + (ngroups ? ngroups + 1 : 0));
    g.atoms.assign(group_atoms, group_atoms + total); g.weight.assign(group_weights, group_weights + total);
    API_END(ctx)
}
extern "C" int b200md_set_custom_globals(b200md_ctx* ctx, int n, const double* values) {
    API_BEGIN(ctx)
    require(n >= 0, "set_custom_globals: negative count");
    CustomTable& t = ctx->custom;
    if (!ctx->finalized) { t.globals.assign(values, values + n); return 0; }
    require(n == (int) t.globals.size(), "set_custom_globals: the number of global parameters cannot change after finalize");
    t.globals.assign(values, values + n);
    // stream ordered, into the buffer the step graphs read: no graph is captured or instantiated again
    if (n) CUDA_CHECK(cudaMemcpyAsync(t.globalsDev.p, t.globals.data(), sizeof(double)*n, cudaMemcpyHostToDevice, ctx->stream));
    API_END(ctx)
}
// The probes: program `which` of a program set of class cls, checked as the set call checks it (nglobals = the number of
// global slots) and run on the host by the interpreter source the device kernels run.  name begins the probe's own messages.
static int custom_probe(const char* name, int cls, int nexpr, const int* nparticles, int periodic, const int* prog_start, const int* op,
                        const int* arg, const double* imm, int stride, int nglobals, int which, const double* vars, const double* box,
                        const double* params, const double* globals, double* out, char* msg, int msglen) {
    try {
        require(nglobals >= 0, (std::string(name) + ": negative number of globals").c_str());
        std::vector<int> exprProg;
        const std::vector<int2> code = check_programs(cls, nexpr, nparticles, prog_start, op, arg, stride, nglobals, exprProg);
        require(which >= 0 && which < exprProg[nexpr], (std::string(name) + ": program index out of range").c_str());
        CustomBox b = {1.0, 0.0, 1.0, 0.0, 0.0, 1.0};
        if (box) b = CustomBox{box[0], box[3], box[4], box[6], box[7], box[8]};
        *out = custom_points(cls)
            ? custom_run<B200MD_CUSTOM_COMPOUND_MAX_STACK, true>(code.data(), imm, prog_start[which], prog_start[which+1], vars, params, globals, b,
                                                                  periodic != 0)
            : custom_run<B200MD_CUSTOM_MAX_STACK, false>(code.data(), imm, prog_start[which], prog_start[which+1], vars, params, globals, b);
        return 0;
    } catch (std::exception& e) {
        if (msg && msglen > 0) { strncpy(msg, e.what(), msglen - 1); msg[msglen - 1] = 0; }
        return -1;
    }
}
extern "C" int b200md_custom_term_probe(int cls, int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                        int stride, int nglobals, int which, const double* vars, const double* box,
                                        const double* params, const double* globals, double* out, char* msg, int msglen) {
    // compound bonds have particle counts: b200md_custom_compound_probe
    if (cls < B200MD_CUSTOM_TORSION || cls > B200MD_CUSTOM_ANGLE) {
        if (msg && msglen > 0) { strncpy(msg, "custom_term_probe: unknown class", msglen - 1); msg[msglen - 1] = 0; }
        return -1;
    }
    return custom_probe("custom_program_probe", cls, nprog, nullptr, 0, prog_start, op, arg, imm, stride, nglobals, which, vars, box, params,
                        globals, out, msg, msglen);
}
extern "C" int b200md_custom_compound_probe(int nparticles, int periodic, const int* prog_start, const int* op, const int* arg, const double* imm,
                                            int stride, int nglobals, int which, const double* vars, const double* box,
                                            const double* params, const double* globals, double* out, char* msg, int msglen) {
    return custom_probe("custom_compound_probe", B200MD_CUSTOM_COMPOUND, 1, &nparticles, periodic, prog_start, op, arg, imm, stride, nglobals,
                        which, vars, box, params, globals, out, msg, msglen);
}
extern "C" int b200md_custom_program_probe(int nprog, const int* prog_start, const int* op, const int* arg, const double* imm,
                                           int stride, int nglobals, int which, double theta, const double* params,
                                           const double* globals, double* out, char* msg, int msglen) {
    return b200md_custom_term_probe(B200MD_CUSTOM_TORSION, nprog, prog_start, op, arg, imm, stride, nglobals, which, &theta, nullptr,
                                    params, globals, out, msg, msglen);
}
extern "C" int b200md_set_bonded_groups(b200md_ctx* ctx, int kind, int n, const int* group) {
    API_BEGIN(ctx)
    check_set(ctx, "set_bonded_groups", n);
    require((kind >= B200MD_BONDED_BONDS && kind <= B200MD_BONDED_CUSTOM_EXTERNALS) || kind == B200MD_BONDED_CUSTOM_ANGLES ||
            kind == B200MD_BONDED_CUSTOM_COMPOUND || kind == B200MD_BONDED_CUSTOM_CENTROID,
            "set_bonded_groups: kind must be 0 (bonds), 1 (angles), 2 (torsions), 3 (RB torsions), 4 (CMAP), 5 (custom torsions), "
            "6 (custom bonds), 7 (custom externals), 9 (custom angles), 10 (custom compound bonds) or 11 (custom centroid bonds)");
    std::vector<unsigned char>* g = kind == B200MD_BONDED_BONDS ? &ctx->bonds.group : kind == B200MD_BONDED_ANGLES ? &ctx->angles.group :
                                    kind == B200MD_BONDED_TORSIONS ? &ctx->torsions.group : kind == B200MD_BONDED_RB_TORSIONS ? &ctx->rb.group :
                                    &ctx->cmap.group;
    for (int k = 0; k < CUSTOM_CLASSES; k++) if (kind == CUSTOM_NAMES[k].kind) g = &ctx->custom.cls[k].group;
    g->resize(n);
    for (int i = 0; i < n; i++) { require(group[i] >= 0 && (group[i] & ~0x80) < 32, "force group out of range"); (*g)[i] = (unsigned char) group[i]; }
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

// The current charges into posq.w (times sqrt(ONE_4PI_EPS0)), positions kept.  Synchronous: the caller has drained the stream.
static void stamp_charges(b200md_ctx* c) {
    const double sk = std::sqrt(B200MD_ONE_4PI_EPS0);
    std::vector<float4> p(c->npad);
    CUDA_CHECK(cudaMemcpy(p.data(), c->posq.p, sizeof(float4)*c->npad, cudaMemcpyDeviceToHost));
    for (int i = 0; i < c->natoms; i++) p[i].w = (float) (c->charge[i]*sk);
    CUDA_CHECK(cudaMemcpy(c->posq.p, p.data(), sizeof(float4)*c->npad, cudaMemcpyHostToDevice));
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
    stamp_charges(c);
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
    require(c->mg == MG_SINGLE, "general (CCMA) constraint networks are not supported in multi-GPU runs");
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
    return c->mg == MG_SINGLE && !c->pmeOnly && c->overlapPme && !c->nb.smPartition && c->nbdesc.method == B200MD_NB_PME;
}

// finalize: the classes of one kernel in its layout: the terms grouped by expression, each group padded to whole warps (a
// padding slot has expression -1 and the atoms `pad`), `width` atoms per slot, the parameters at one stride (the widest
// class's); the expressions and programs of all its classes one after the other (class k's expression p is expression
// exprBase[k] + p), the programs checked once more now that the number of global slots is final.  Returns the term bits of
// the classes that have terms.
static int layout_custom(b200md_ctx* c, CustomSlots& s, int width, int pad) {
    CustomTable& t = c->custom;
    std::vector<int2> code; std::vector<double> imm;
    std::vector<int> progStart(1, 0), exprClass, exprParticles, exprPeriodic, exprProg, exprBase(CUSTOM_CLASSES, 0);
    int terms = 0;
    s.nslots = 0; s.stride = 0;
    for (int k = s.first; k < s.last; k++) {
        const CustomClass& cl = t.cls[k];
        exprBase[k] = (int) exprClass.size();
        if (cl.n == 0) continue;
        require(c->mg == MG_SINGLE, (std::string(CUSTOM_NAMES[k].term) + "s are not supported in multi-GPU runs").c_str());
        require(cl.group.empty() || (int) cl.group.size() == cl.n, "set_bonded_groups: group array length differs from the number of terms");
        std::vector<int> unused;
        const std::vector<int2> cc = check_programs(k, cl.nexpr, cl.nparticles.data(), cl.progStart.data(), cl.op.data(), cl.arg.data(), cl.stride,
                                                    (int) t.globals.size(), unused);
        const int progBase = (int) progStart.size() - 1, codeBase = (int) code.size();
        for (int p = 0; p < cl.nexpr; p++) {
            exprClass.push_back(k); exprParticles.push_back(cl.nparticles[p]); exprPeriodic.push_back(cl.periodic[p]);
            exprProg.push_back(progBase + cl.exprProg[p]);
        }
        for (int q = 0; q < cl.exprProg[cl.nexpr]; q++) progStart.push_back(codeBase + cl.progStart[q+1]);
        code.insert(code.end(), cc.begin(), cc.end());
        imm.insert(imm.end(), cl.imm.begin(), cl.imm.end());
        s.stride = std::max(s.stride, cl.stride);
        terms |= CUSTOM_NAMES[k].bit;
    }
    if (terms == 0) return 0;
    int cursor = 0;
    for (int k = s.first; k < s.last; k++) {
        CustomClass& cl = t.cls[k];
        cl.slot.assign(cl.n, 0);
        for (int p = 0; p < cl.nexpr; p++) {
            for (int i = 0; i < cl.n; i++) if (cl.expr[i] == p) cl.slot[i] = cursor++;
            cursor = (cursor + 31)/32*32;
        }
    }
    s.nslots = cursor;
    std::vector<int> atoms((size_t) width*cursor, pad), expr(cursor, -1);
    std::vector<unsigned char> group(cursor, 0);
    for (int k = s.first; k < s.last; k++) {
        const CustomClass& cl = t.cls[k];
        const int w = CUSTOM_NAMES[k].width;
        for (int i = 0; i < cl.n; i++) {
            std::copy(cl.atoms.begin() + (size_t) w*i, cl.atoms.begin() + (size_t) w*(i+1), atoms.begin() + (size_t) width*cl.slot[i]);
            group[cl.slot[i]] = cl.group.empty() ? 0 : cl.group[i]; expr[cl.slot[i]] = exprBase[k] + cl.expr[i];
        }
    }
    s.atomsDev.upload(atoms); s.groupDev.upload(group); s.exprDev.upload(expr);
    const std::vector<double> par = t.slot_params(s);
    s.paramsDev.alloc(std::max<size_t>(par.size(), 1)); s.paramsDev.upload(par);
    s.codeDev.upload(code); s.immDev.upload(imm); s.progStartDev.upload(progStart);
    s.exprClassDev.upload(exprClass); s.exprParticlesDev.upload(exprParticles); s.exprPeriodicDev.upload(exprPeriodic); s.exprProgDev.upload(exprProg);
    return terms;
}

// finalize: the classes of s in the layout of k_compound (CompoundDev: 8 atoms, or groups, per slot, unused -1)
static void layout_compound(b200md_ctx* c, CustomSlots& u, CompoundDev& e) {
    e = CompoundDev{};
    e.groupMask = 0xffffffffu;
    e.globals = c->custom.globalsDev.p;
    layout_custom(c, u, B200MD_CUSTOM_MAX_PARTICLES, -1);
    e.nslots = u.nslots; e.paramStride = u.stride;
    e.atoms = u.atomsDev.p; e.params = u.paramsDev.p; e.group = u.groupDev.p; e.expr = u.exprDev.p;
    e.exprParticles = u.exprParticlesDev.p; e.exprPeriodic = u.exprPeriodicDev.p; e.exprProg = u.exprProgDev.p;
    e.code = u.codeDev.p; e.imm = u.immDev.p; e.progStart = u.progStartDev.p;
}

// finalize: the centroid bonds' groups (CentroidDev): the CSR, room for the centres and the derivatives of every slot, and
// the scatter entries in slot order, (slot, group position k, atom) of every atom of weight != 0 of every group of every term
static void upload_centroid(b200md_ctx* c) {
    CustomTable& t = c->custom;
    CentroidGroups& g = t.groups;
    CentroidDev& d = c->cen;
    d = CentroidDev{};
    if (c->ccd.nslots == 0) return;
    const CustomClass& cl = t.cls[B200MD_CUSTOM_CENTROID];
    const int nslots = c->ccd.nslots;
    std::vector<int> termOf(nslots, -1);
    for (int i = 0; i < cl.n; i++) termOf[cl.slot[i]] = i;
    std::vector<int4> scatter; std::vector<double> weight;
    for (int s = 0; s < nslots; s++) {
        const int i = termOf[s];
        if (i < 0) continue;
        for (int k = 0; k < cl.nparticles[cl.expr[i]]; k++) {
            const int grp = cl.atoms[B200MD_CUSTOM_MAX_PARTICLES*(size_t) i + k];
            for (int a = g.start[grp]; a < g.start[grp+1]; a++)
                if (g.weight[a] != 0.0) { scatter.push_back(make_int4(s, k, g.atoms[a], 0)); weight.push_back(g.weight[a]); }
        }
    }
    const int ngroups = (int) g.start.size() - 1;
    g.startDev.upload(g.start); g.atomsDev.upload(g.atoms); g.weightDev.upload(g.weight);
    g.centerDev.alloc(3*(size_t) ngroups); g.centerDev.zero();
    g.derivDev.alloc((size_t) nslots*CENTROID_DERIVS); g.derivDev.zero();
    g.scatterDev.upload(scatter); g.scatterWeightDev.upload(weight);
    d.ngroups = ngroups; d.nscatter = (int) scatter.size();
    d.groupStart = g.startDev.p; d.groupAtoms = g.atomsDev.p; d.groupWeight = g.weightDev.p;
    d.center = g.centerDev.p; d.deriv = g.derivDev.p;
    d.scatter = g.scatterDev.p; d.scatterWeight = g.scatterWeightDev.p;
}

// finalize: the custom terms in the layouts of k_custom (CustomDev: int4 atoms, zero-padded) and k_compound (CompoundDev: 8
// atoms per slot, unused -1; the centroid bonds in a second one), and the global values all read
static void upload_custom(b200md_ctx* c) {
    CustomTable& t = c->custom;
    // the global values get their buffer even without terms: a custom force with no terms may still name globals, and
    // b200md_set_custom_globals copies into this buffer after finalize
    t.globalsDev.alloc(std::max<size_t>(t.globals.size(), 1)); t.globalsDev.upload(t.globals);
    CustomSlots& s = t.kernel[0];
    CustomDev& d = c->ctd;
    d = CustomDev{};
    d.groupMask = 0xffffffffu;
    d.globals = t.globalsDev.p;
    d.terms = layout_custom(c, s, 4, 0);
    d.nslots = s.nslots; d.paramStride = s.stride;
    d.atoms = (const int4*) s.atomsDev.p; d.params = s.paramsDev.p; d.group = s.groupDev.p; d.expr = s.exprDev.p;
    d.exprClass = s.exprClassDev.p; d.exprProg = s.exprProgDev.p;
    d.code = s.codeDev.p; d.imm = s.immDev.p; d.progStart = s.progStartDev.p;
    layout_compound(c, t.kernel[1], c->cpd);
    layout_compound(c, t.kernel[2], c->ccd);
    upload_centroid(c);
}

extern "C" int b200md_finalize(b200md_ctx* ctx) {
    API_BEGIN(ctx)
    require(!ctx->finalized, "finalize called twice");
    b200md_ctx* c = ctx;
    const int N = c->natoms, NP = c->npad;
    if (!c->haveNb) {
        // no NonbondedForce: the list is built for the custom nonbonded force alone, at its method and cutoff
        c->nbdesc = b200md_nonbonded_desc{};
        c->nbdesc.method = c->cnb.have ? c->cnb.method : B200MD_NB_NOCUTOFF;
        if (c->cnb.have) c->nbdesc.cutoff = c->cnb.cutoff;
    }
    NbDev& nb = c->nb;
    nb.natoms = N; nb.npad = NP; nb.nblocks = c->nblocks;
    nb.method = c->nbdesc.method;
    const bool nccl = getenv("B200MD_MGPU") && std::string(getenv("B200MD_MGPU")) == "nccl";
    // b200md_comm_init sets world and comm together
    c->mg = c->world == 1 ? MG_SINGLE : !nccl ? MG_P2P : (nb.method == B200MD_NB_PME && c->haveNb) ? MG_NCCL_SPLIT : MG_NCCL_SHARED;
    // this rank's share of the sharded kernels (k_bonded, k_build_tiles, k_pair, the user-order k_pme_spread and
    // k_pme_gather): in the NCCL role split the PME rank takes every atom, the direct ranks deal the rest among world-1
    nb.rank = c->rank; nb.world = c->world;
    if (c->mg == MG_NCCL_SPLIT) {
        if (c->rank == c->world - 1) { nb.rank = 0; nb.world = 1; }
        else nb.world = c->world - 1;
    }
    c->cd = CommDev{}; c->cd.world = 1;
    if (c->mg == MG_P2P) setup_window(c);
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
        if (c->mg == MG_P2P) want = std::min(74, std::max((c->nbdesc.grid[0] + c->world - 1)/c->world, 16 + 6*c->world));
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
        if (!c->haveNb) for (const int2& a : c->cnb.excl) { ex[a.x].push_back(a.y); ex[a.y].push_back(a.x); }
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
    upload_custom(c);
    upload_params(c);
    build_units(c);
    build_ccma(c);
    setup_gbsa(c);
    setup_custom_nonbonded(c);
    setup_rmsd(c);
    setup_cv(c);
    if (c->mg == MG_P2P) {
        setup_ownership(c);
        if (nb.method == B200MD_NB_PME) {
            PmeDev probe{}; probe.nx = c->nbdesc.grid[0]; probe.ny = c->nbdesc.grid[1]; probe.nz = c->nbdesc.grid[2]; probe.nzc = probe.nz/2 + 1;
            require(fft_slab_path(probe), "multi-GPU: the PME grid plane does not fit the slab FFT kernels (B200MD_MGPU=nccl selects the NCCL scheme)");
        }
    }
    // ---- molecules (connected components of bonds, angles, torsions, RB torsions, CMAP terms, custom torsions, bonds and
    // angles, constraints and exceptions; not custom externals, which act on one particle, nor custom compound and centroid
    // bonds, which read continuous coordinates and may tie two molecules that must keep wrapping apart) for the wrap at list
    // builds; off for non-periodic systems and with more than one rank (every rank would have to wrap in the same step,
    // and the reciprocal-space rank builds no list) ----
    c->cellOffset.alloc((size_t) 3*NP); c->cellOffset.zero();
    nb.cellOffset = c->cellOffset.p; nb.nmol = 0; nb.molStart = nullptr; nb.molAtoms = nullptr;
    if ((nb.method == B200MD_NB_CUTOFF_PERIODIC || nb.method == B200MD_NB_PME) && c->mg == MG_SINGLE && !c->pmeOnly) {
        std::vector<int> parent(N);
        for (int i = 0; i < N; i++) parent[i] = i;
        auto find = [&](int x) { while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; } return x; };
        auto join = [&](int a, int b) { a = find(a); b = find(b); if (a != b) parent[std::max(a, b)] = std::min(a, b); };
        for (const int2& a : c->bonds.atoms) join(a.x, a.y);
        for (const int4& a : c->angles.atoms) { join(a.x, a.y); join(a.y, a.z); }
        for (auto* t : {&c->torsions.atoms, &c->rb.atoms, &c->cmap.atoms}) for (const int4& a : *t) { join(a.x, a.y); join(a.y, a.z); join(a.z, a.w); }
        for (int k = 0; k < CUSTOM_CLASSES; k++) {
            const CustomClass& cl = c->custom.cls[k];
            const int w = CUSTOM_NAMES[k].width;
            if (CUSTOM_NAMES[k].joins)
                for (int i = 0; i < cl.n; i++) for (int j = 1; j < w; j++) join(cl.atoms[w*i + j - 1], cl.atoms[w*i + j]);
        }
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

// CalcCustom{Torsion,Bond,External,Angle,CompoundBond,CentroidBond}ForceKernel::copyParametersToContext (kernels.h): same terms and
// programs, new parameters, into the same device buffer.
static void update_custom(b200md_ctx* ctx, int cls, int n, const double* params) {
    const CustomNames& nm = CUSTOM_NAMES[cls];
    require(ctx->finalized, (std::string(nm.update) + " before finalize").c_str());
    CustomTable& t = ctx->custom;
    CustomClass& cl = t.cls[cls];
    require(n == cl.n, (std::string("updateParametersInContext: The number of ") + nm.terms + " has changed").c_str());
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    cl.params.assign(params, params + (size_t) n*cl.stride);
    CustomSlots& s = t.kernel_of(cls);
    if (n) s.paramsDev.upload(t.slot_params(s));
}
extern "C" int b200md_update_custom_torsion_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    update_custom(ctx, B200MD_CUSTOM_TORSION, n, params);
    API_END(ctx)
}
extern "C" int b200md_update_custom_bond_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    update_custom(ctx, B200MD_CUSTOM_BOND, n, params);
    API_END(ctx)
}
extern "C" int b200md_update_custom_external_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    update_custom(ctx, B200MD_CUSTOM_EXTERNAL, n, params);
    API_END(ctx)
}
extern "C" int b200md_update_custom_angle_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    update_custom(ctx, B200MD_CUSTOM_ANGLE, n, params);
    API_END(ctx)
}
extern "C" int b200md_update_custom_compound_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    update_custom(ctx, B200MD_CUSTOM_COMPOUND, n, params);
    API_END(ctx)
}
extern "C" int b200md_update_custom_centroid_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    update_custom(ctx, B200MD_CUSTOM_CENTROID, n, params);
    API_END(ctx)
}

// ---------------------------------------------------------------- CustomNonbondedForce
// The programs of nobj objects, 2 each (energy, dE/dr), every one passing custom_check_program for its object's nparams[o] <=
// B200MD_CUSTOM_MAX_PARAMS/2 parameters per particle (nglobals, ntables < 0: checked at finalize).  Returns the instructions.
static std::vector<int2> check_nonbonded_programs(const std::string& call, int nobj, const int* prog_start, const int* op, const int* arg,
                                                  const int* nparams, int nglobals, int ntables) {
    require(nobj >= 1, (call + ": at least one object").c_str());
    require(prog_start[0] == 0, (call + ": prog_start[0] must be 0").c_str());
    for (int q = 0; q < 2*nobj; q++) require(prog_start[q+1] >= prog_start[q], (call + ": prog_start must not decrease").c_str());
    std::vector<int2> code(prog_start[2*nobj]);
    for (size_t k = 0; k < code.size(); k++) code[k] = make_int2(op[k], arg[k]);
    for (int o = 0; o < nobj; o++) {
        require(nparams[o] >= 0 && nparams[o] <= B200MD_CUSTOM_MAX_PARAMS/2, (call + ": more than 8 per-particle parameters").c_str());
        for (int q = 2*o; q < 2*o + 2; q++) {
            const char* why = custom_check_program(B200MD_CUSTOM_NONBONDED, code.data(), prog_start[q], prog_start[q+1], 2*nparams[o], nglobals, 0, ntables);
            if (why) throw std::runtime_error(std::string(why) + " (program " + std::to_string(q) + ")");
        }
    }
    return code;
}
// ntables tables: 1 to 3 dimensions of at least one entry each (unused ones 1), start[t+1] - start[t] entries each
static void check_tables(const std::string& call, int ntables, const int* dims, const int* start) {
    require(ntables >= 0, (call + ": negative number of tables").c_str());
    require(ntables == 0 || start[0] == 0, (call + ": start[0] must be 0").c_str());
    for (int t = 0; t < ntables; t++) {
        const int nd = dims[4*t];
        require(nd >= 1 && nd <= 3, (call + ": a table has 1, 2 or 3 dimensions").c_str());
        long long size = 1;
        for (int k = 0; k < 3; k++) {
            require(dims[4*t + 1 + k] >= 1 && (k < nd || dims[4*t + 1 + k] == 1), (call + ": a table size must be at least 1 (1 for an unused dimension)").c_str());
            size *= dims[4*t + 1 + k];
        }
        require(start[t+1] - start[t] == size, (call + ": a table's number of values does not match its sizes").c_str());
    }
}
static void check_cnb_params(const b200md_ctx* c, const char* call, int nobj, int stride, const double* params) {
    for (size_t k = 0; k < (size_t) nobj*c->natoms*stride; k++)
        require(std::isfinite(params[k]), (std::string(call) + ": a per-particle parameter is not finite").c_str());
}
extern "C" int b200md_set_custom_nonbonded(b200md_ctx* ctx, int method, double cutoff, int nobj, const int* prog_start, const int* op, const int* arg,
                                           const double* imm, const int* nparams, int stride, const double* params,
                                           const double* switch_distance, const int* group, int nexcl, const int* excl_p1, const int* excl_p2) {
    API_BEGIN(ctx)
    check_set(ctx, "set_custom_nonbonded", nobj);
    check_set(ctx, "set_custom_nonbonded", nexcl);
    require(ctx->world == 1, "CustomNonbondedForce is not supported in multi-GPU runs");
    require(method == B200MD_NB_NOCUTOFF || method == B200MD_NB_CUTOFF_NONPERIODIC || method == B200MD_NB_CUTOFF_PERIODIC,
            "set_custom_nonbonded: method must be NoCutoff, CutoffNonPeriodic or CutoffPeriodic");
    require(method == B200MD_NB_NOCUTOFF || (std::isfinite(cutoff) && cutoff > 0.0), "set_custom_nonbonded: the cutoff must be positive");
    require(stride >= 0 && stride <= B200MD_CUSTOM_MAX_PARAMS/2, "set_custom_nonbonded: more than 8 per-particle parameters");
    const std::vector<int2> code = check_nonbonded_programs("set_custom_nonbonded", nobj, prog_start, op, arg, nparams, -1, -1);
    for (int o = 0; o < nobj; o++) {
        require(nparams[o] <= stride, "set_custom_nonbonded: an object has more parameters than param_stride");
        const double sw = switch_distance[o];
        require(sw < 0.0 || (method != B200MD_NB_NOCUTOFF && sw < cutoff), "set_custom_nonbonded: the switching distance must be below the cutoff");
        require(group[o] >= 0 && group[o] < 32, "set_custom_nonbonded: force group out of range");
    }
    for (int k = 0; k < nexcl; k++)
        require(excl_p1[k] >= 0 && excl_p1[k] < ctx->natoms && excl_p2[k] >= 0 && excl_p2[k] < ctx->natoms && excl_p1[k] != excl_p2[k],
                "set_custom_nonbonded: an excluded pair must be two different particles");
    check_cnb_params(ctx, "set_custom_nonbonded", nobj, stride, params);
    auto& g = ctx->cnb;
    g.have = true; g.method = method; g.cutoff = method == B200MD_NB_NOCUTOFF ? 0.0 : cutoff; g.nobj = nobj; g.stride = stride;
    const int total = prog_start[2*nobj];
    g.progStart.assign(prog_start, prog_start + 2*nobj + 1);
    g.op.assign(op, op + total); g.arg.assign(arg, arg + total); g.imm.assign(imm, imm + total);
    g.nparams.assign(nparams, nparams + nobj); g.group.assign(group, group + nobj);
    g.switchDist.assign(switch_distance, switch_distance + nobj);
    g.params.assign(params, params + (size_t) nobj*ctx->natoms*stride);
    g.lrc.assign(nobj, 0.0);
    g.excl.resize(nexcl);
    for (int k = 0; k < nexcl; k++) g.excl[k] = make_int2(excl_p1[k], excl_p2[k]);
    API_END(ctx)
}
extern "C" int b200md_set_custom_tables(b200md_ctx* ctx, int ntables, const int* dims, const int* start, const double* values) {
    API_BEGIN(ctx)
    check_set(ctx, "set_custom_tables", ntables);
    check_tables("set_custom_tables", ntables, dims, start);
    auto& g = ctx->cnb;
    g.tableDims.resize(ntables);
    for (int t = 0; t < ntables; t++) g.tableDims[t] = make_int4(dims[4*t], dims[4*t + 1], dims[4*t + 2], dims[4*t + 3]);
    g.tableStart.assign(start, start + ntables + 1);
    g.tableValues.assign(values, values + (ntables ? start[ntables] : 0));
    API_END(ctx)
}
// the parameters of every object, [nobj][npad][stride] (padding atoms 0), into buffers of a fixed size: a captured step graph
// keeps its pointers
static void upload_cnb_params(b200md_ctx* c) {
    auto& g = c->cnb;
    const int st = std::max(g.stride, 1);
    std::vector<double> p((size_t) g.nobj*c->npad*st, 0.0);
    for (int o = 0; o < g.nobj; o++)
        for (int i = 0; i < c->natoms; i++)
            for (int k = 0; k < g.stride; k++) p[((size_t) o*c->npad + i)*st + k] = g.params[((size_t) o*c->natoms + i)*g.stride + k];
    g.paramsDev.upload(p);
}
extern "C" int b200md_update_custom_nonbonded_params(b200md_ctx* ctx, int n, const double* params) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_custom_nonbonded_params before finalize");
    require(ctx->cnb.have, "update_custom_nonbonded_params: the context has no custom nonbonded force");
    require(n == ctx->natoms, "update_custom_nonbonded_params: the number of particles has changed");
    auto& g = ctx->cnb;
    check_cnb_params(ctx, "update_custom_nonbonded_params", g.nobj, g.stride, params);
    g.params.assign(params, params + (size_t) g.nobj*n*g.stride);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    upload_cnb_params(ctx);
    API_END(ctx)
}
extern "C" int b200md_set_custom_nonbonded_lrc(b200md_ctx* ctx, int nobj, const double* coefficient) {
    API_BEGIN(ctx)
    require(ctx->cnb.have && nobj == ctx->cnb.nobj, "set_custom_nonbonded_lrc: one coefficient per custom nonbonded object");
    for (int o = 0; o < nobj; o++) require(std::isfinite(coefficient[o]), "set_custom_nonbonded_lrc: a coefficient is not finite");
    ctx->cnb.lrc.assign(coefficient, coefficient + nobj);
    API_END(ctx)
}
// finalize: the method, cutoff and exclusions must be the list's (those of the nonbonded force, when there is one), the
// programs' global and table operands in range; the device state and the stream
static void setup_custom_nonbonded(b200md_ctx* c) {
    auto& g = c->cnb;
    c->cnd = CnbDev{};
    if (!g.have) return;
    require(c->world == 1, "CustomNonbondedForce is not supported in multi-GPU runs");
    if (c->haveNb) {
        const int nm = c->nbdesc.method;
        require(g.method == B200MD_NB_CUTOFF_PERIODIC ? (nm == B200MD_NB_CUTOFF_PERIODIC || nm == B200MD_NB_PME) : nm == g.method,
                "custom nonbonded force: its method does not match the nonbonded force's (CutoffPeriodic goes with CutoffPeriodic or PME)");
        if (g.method != B200MD_NB_NOCUTOFF)
            require(std::fabs(g.cutoff - c->nbdesc.cutoff) <= 1e-12*c->nbdesc.cutoff, "custom nonbonded force: the cutoff must be that of the nonbonded force");
        auto pairs = [](const std::vector<int2>& v) {
            std::vector<std::pair<int, int> > p;
            for (const int2& a : v) p.push_back(std::make_pair(std::min(a.x, a.y), std::max(a.x, a.y)));
            std::sort(p.begin(), p.end());
            p.erase(std::unique(p.begin(), p.end()), p.end());
            return p;
        };
        require(pairs(g.excl) == pairs(c->exc.atoms), "custom nonbonded force: its exclusions must be the nonbonded force's exceptions");
    }
    const int ntables = (int) g.tableDims.size();
    check_nonbonded_programs("custom nonbonded force", g.nobj, g.progStart.data(), g.op.data(), g.arg.data(), g.nparams.data(),
                             (int) c->custom.globals.size(), ntables);
    std::vector<int2> code(g.op.size());
    for (size_t k = 0; k < code.size(); k++) code[k] = make_int2(g.op[k], g.arg[k]);
    g.codeDev.upload(code); g.immDev.upload(g.imm); g.progStartDev.upload(g.progStart);
    g.nparamsDev.upload(g.nparams); g.groupDev.upload(g.group); g.switchDev.upload(g.switchDist);
    upload_cnb_params(c);
    g.tableDimsDev.alloc(std::max(ntables, 1)); g.tableDimsDev.upload(g.tableDims);
    g.tableStartDev.alloc(ntables + 1); g.tableStartDev.upload(ntables ? g.tableStart : std::vector<int>(1, 0));
    g.tableValuesDev.alloc(std::max<size_t>(g.tableValues.size(), 1)); g.tableValuesDev.upload(g.tableValues);
    CnbDev& d = c->cnd;
    d.nobj = g.nobj; d.stride = std::max(g.stride, 1);
    d.useCutoff = g.method != B200MD_NB_NOCUTOFF;
    d.cutoff = g.cutoff; d.cutoff2 = g.cutoff*g.cutoff;
    d.nparams = g.nparamsDev.p; d.switchDist = g.switchDev.p; d.group = g.groupDev.p; d.params = g.paramsDev.p;
    d.code = g.codeDev.p; d.imm = g.immDev.p; d.progStart = g.progStartDev.p;
    d.globals = c->custom.globalsDev.p;
    d.ntables = ntables; d.tableDims = g.tableDimsDev.p; d.tableStart = g.tableStartDev.p; d.tableValues = g.tableValuesDev.p;
    d.groupMask = 0xffffffffu;
    if (!g.stream) {
        int hi = 0;
        CUDA_CHECK(cudaDeviceGetStreamPriorityRange(nullptr, &hi));
        CUDA_CHECK(cudaStreamCreateWithPriority(&g.stream, cudaStreamNonBlocking, hi));
        CUDA_CHECK(cudaEventCreateWithFlags(&g.evFork, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&g.evJoin, cudaEventDisableTiming));
    }
}
extern "C" int b200md_custom_nonbonded_probe(int nprog, const int* prog_start, const int* op, const int* arg, const double* imm, int nparams,
                                             int nglobals, int which, double r, const double* params, const double* globals, int ntables,
                                             const int* dims, const int* start, const double* values, double* out, char* msg, int msglen) {
    try {
        require(nprog >= 2 && nprog % 2 == 0, "custom_nonbonded_probe: two programs per object");
        require(nglobals >= 0, "custom_nonbonded_probe: negative number of globals");
        check_tables("custom_nonbonded_probe", ntables, dims, start);
        const std::vector<int> np(nprog/2, nparams);
        const std::vector<int2> code = check_nonbonded_programs("custom_nonbonded_probe", nprog/2, prog_start, op, arg, np.data(), nglobals, ntables);
        require(which >= 0 && which < nprog, "custom_nonbonded_probe: program index out of range");
        std::vector<int4> d(ntables);
        for (int t = 0; t < ntables; t++) d[t] = make_int4(dims[4*t], dims[4*t + 1], dims[4*t + 2], dims[4*t + 3]);
        const CustomTables tables = {ntables, d.data(), start, values};
        const CustomBox b = {1.0, 0.0, 1.0, 0.0, 0.0, 1.0};
        *out = custom_run<B200MD_CUSTOM_MAX_STACK, false, true>(code.data(), imm, prog_start[which], prog_start[which+1], &r, params, globals, b,
                                                                 false, &tables);
        return 0;
    } catch (std::exception& e) {
        if (msg && msglen > 0) { strncpy(msg, e.what(), msglen - 1); msg[msglen - 1] = 0; }
        return -1;
    }
}

// ---------------------------------------------------------------- generalized Born (GBSAOBCForce)
// charge, radius and scale of every atom: finite, radius above the dielectric offset (ObcParameters' rho = R - 0.009 must be
// positive), scale not negative
static void check_gbsa_params(const b200md_ctx* c, const char* call, const double* q, const double* r, const double* s) {
    for (int i = 0; i < c->natoms; i++) {
        require(std::isfinite(q[i]) && std::isfinite(r[i]) && std::isfinite(s[i]), (std::string(call) + ": a parameter is not finite").c_str());
        require(r[i] > 0.009, (std::string(call) + ": a radius must exceed the dielectric offset of 0.009 nm").c_str());
        require(s[i] >= 0.0, (std::string(call) + ": a scale factor must not be negative").c_str());
    }
}
// the device form of the per-atom parameters (GbsaDev), into buffers of a fixed size: a captured step graph keeps its pointers
static void upload_gbsa_params(b200md_ctx* c) {
    const int N = c->natoms;
    std::vector<float> q(c->npad, 0.f); std::vector<double2> rad(c->npad, make_double2(1.0, 0.0)); std::vector<double> R(c->npad, 1.0);
    for (int i = 0; i < N; i++) {
        const double rho = c->gbsa.radius[i] - 0.009;
        q[i] = (float) (c->gbsa.charge[i]*std::sqrt(B200MD_ONE_4PI_EPS0));
        rad[i] = make_double2(rho, rho*c->gbsa.scale[i]);
        R[i] = c->gbsa.radius[i];
    }
    c->gbsa.chargeDev.upload(q); c->gbsa.radiusDev.upload(rad); c->gbsa.atomRadiusDev.upload(R);
}
extern "C" int b200md_set_gbsa(b200md_ctx* ctx, int method, double cutoff, double solute, double solvent, double surface,
                               const double* charge, const double* radius, const double* scale) {
    API_BEGIN(ctx)
    check_set(ctx, "set_gbsa", 0);
    require(ctx->world == 1, "generalized Born (GBSAOBCForce) is not supported in multi-GPU runs");
    require(method == B200MD_NB_NOCUTOFF || method == B200MD_NB_CUTOFF_NONPERIODIC || method == B200MD_NB_CUTOFF_PERIODIC,
            "set_gbsa: method must be NoCutoff, CutoffNonPeriodic or CutoffPeriodic");
    require(method == B200MD_NB_NOCUTOFF || (std::isfinite(cutoff) && cutoff > 0.0), "set_gbsa: the cutoff must be positive");
    require(std::isfinite(solute) && std::isfinite(solvent) && std::isfinite(surface), "set_gbsa: the dielectrics and the surface energy must be finite");
    check_gbsa_params(ctx, "set_gbsa", charge, radius, scale);
    auto& g = ctx->gbsa;
    g.have = true; g.method = method; g.cutoff = cutoff; g.solute = solute; g.solvent = solvent; g.surface = surface;
    g.charge.assign(charge, charge + ctx->natoms); g.radius.assign(radius, radius + ctx->natoms); g.scale.assign(scale, scale + ctx->natoms);
    API_END(ctx)
}
extern "C" int b200md_update_gbsa_params(b200md_ctx* ctx, int n, const double* charge, const double* radius, const double* scale) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_gbsa_params before finalize");
    require(ctx->gbsa.have, "update_gbsa_params: the context has no generalized Born force");
    require(n == ctx->natoms, "update_gbsa_params: the number of particles has changed");
    check_gbsa_params(ctx, "update_gbsa_params", charge, radius, scale);
    auto& g = ctx->gbsa;
    g.charge.assign(charge, charge + n); g.radius.assign(radius, radius + n); g.scale.assign(scale, scale + n);
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    upload_gbsa_params(ctx);
    API_END(ctx)
}
// finalize: the method must agree with the nonbonded one (the chain walks its list), the device state, and the stream
static void setup_gbsa(b200md_ctx* c) {
    auto& g = c->gbsa;
    c->gbd = GbsaDev{};
    if (!g.have) return;
    require(c->world == 1, "generalized Born (GBSAOBCForce) is not supported in multi-GPU runs");
    const int nm = c->haveNb ? c->nbdesc.method : -1;
    // without a nonbonded force the list is the custom nonbonded force's: the chain needs it to hold every pair
    if (!c->haveNb && c->cnb.have)
        require(c->cnb.method == B200MD_NB_NOCUTOFF, "generalized Born at NoCutoff beside a custom nonbonded force with a cutoff needs a nonbonded force");
    if (!c->haveNb) require(g.method == B200MD_NB_NOCUTOFF, "generalized Born with a cutoff needs a nonbonded force with the same cutoff");
    else if (g.method == B200MD_NB_NOCUTOFF) require(nm == B200MD_NB_NOCUTOFF, "generalized Born: NoCutoff needs a NoCutoff nonbonded force");
    else if (g.method == B200MD_NB_CUTOFF_NONPERIODIC) require(nm == B200MD_NB_CUTOFF_NONPERIODIC, "generalized Born: CutoffNonPeriodic needs a CutoffNonPeriodic nonbonded force");
    else require(nm == B200MD_NB_CUTOFF_PERIODIC || nm == B200MD_NB_PME, "generalized Born: CutoffPeriodic needs a CutoffPeriodic or PME nonbonded force");
    if (g.method != B200MD_NB_NOCUTOFF)
        require(std::fabs(g.cutoff - c->nbdesc.cutoff) <= 1e-12*c->nbdesc.cutoff, "generalized Born: the cutoff must be that of the nonbonded force");
    upload_gbsa_params(c);
    const int NP = c->npad;
    g.bornSum.alloc(NP); g.bornSum.zero(); g.dEdB.alloc(NP); g.dEdB.zero();
    g.bornR.alloc(NP); g.bornR.zero(); g.chain.alloc(NP); g.chain.zero(); g.bornForce.alloc(NP); g.bornForce.zero();
    GbsaDev& d = c->gbd;
    d.useCutoff = g.method != B200MD_NB_NOCUTOFF;
    d.cutoff = d.useCutoff ? g.cutoff : 0.0; d.cutoff2 = d.cutoff*d.cutoff;
    d.prefactor = (g.solute != 0.0 && g.solvent != 0.0) ? -(1.0/g.solute - 1.0/g.solvent) : 0.0;
    d.surfaceFactor = 4.0*M_PI*g.surface;
    d.charge = g.chargeDev.p; d.radius = g.radiusDev.p; d.atomRadius = g.atomRadiusDev.p;
    d.bornSum = g.bornSum.p; d.dEdB = g.dEdB.p; d.bornR = g.bornR.p; d.chain = g.chain.p; d.bornForce = g.bornForce.p;
    if (!g.stream) {
        int hi = 0;
        CUDA_CHECK(cudaDeviceGetStreamPriorityRange(nullptr, &hi));
        CUDA_CHECK(cudaStreamCreateWithPriority(&g.stream, cudaStreamNonBlocking, hi));
        CUDA_CHECK(cudaEventCreateWithFlags(&g.evFork, cudaEventDisableTiming));
        CUDA_CHECK(cudaEventCreateWithFlags(&g.evJoin, cudaEventDisableTiming));
    }
}

// ---------------------------------------------------------------- RMSDForce
// nforces objects: object o is the particles particles[start[o] .. start[o+1]-1] (at least one, each at most once, in range)
// with the reference positions ref[3 k ..] of entry k; kept on the host with every reference position centred over its object
static void read_rmsd(b200md_ctx* c, const char* call, int nforces, const int* start, const int* particles, const double* ref) {
    require(nforces >= 0, (std::string(call) + ": negative count").c_str());
    require(nforces == 0 || start[0] == 0, (std::string(call) + ": start[0] must be 0").c_str());
    auto& r = c->rmsd;
    std::vector<int> st(start, start + nforces + 1), atoms, obj;
    std::vector<double> pos, sq;
    for (int o = 0; o < nforces; o++) {
        require(st[o+1] > st[o], (std::string(call) + ": an RMSD force has no particles").c_str());
        std::set<int> seen;
        double cen[3] = {0.0, 0.0, 0.0};
        for (int k = st[o]; k < st[o+1]; k++) {
            const int a = particles[k];
            require(a >= 0 && a < c->natoms, (std::string(call) + ": particle index out of range").c_str());
            require(seen.insert(a).second, (std::string(call) + ": a particle appears twice in one RMSD force").c_str());
            for (int d = 0; d < 3; d++) {
                require(std::isfinite(ref[3*k + d]), (std::string(call) + ": a reference position is not finite").c_str());
                cen[d] += ref[3*k + d];
            }
        }
        const int n = st[o+1] - st[o];
        double s2 = 0.0;
        for (int k = st[o]; k < st[o+1]; k++) {
            atoms.push_back(particles[k]); obj.push_back(o);
            for (int d = 0; d < 3; d++) { const double x = ref[3*k + d] - cen[d]/n; pos.push_back(x); s2 += x*x; }
        }
        sq.push_back(s2);
    }
    r.start.swap(st); r.atoms.swap(atoms); r.entryObj.swap(obj); r.ref.swap(pos); r.refSq.swap(sq);
}
static void upload_rmsd(b200md_ctx* c) {
    auto& r = c->rmsd;
    r.startDev.upload(r.start); r.atomsDev.upload(r.atoms); r.entryObjDev.upload(r.entryObj); r.refDev.upload(r.ref); r.refSqDev.upload(r.refSq);
}
extern "C" int b200md_set_rmsd(b200md_ctx* ctx, int nforces, const int* start, const int* particles, const double* ref, const int* group) {
    API_BEGIN(ctx)
    check_set(ctx, "set_rmsd", nforces);
    require(ctx->world == 1, "RMSDForce is not supported in multi-GPU runs");
    read_rmsd(ctx, "set_rmsd", nforces, start, particles, ref);
    ctx->rmsd.group.assign(nforces, 0);
    for (int o = 0; o < nforces; o++) {
        require(group[o] >= 0 && group[o] <= 31, "set_rmsd: force group out of range");
        ctx->rmsd.group[o] = (unsigned char) group[o];
    }
    API_END(ctx)
}
extern "C" int b200md_update_rmsd(b200md_ctx* ctx, int nforces, const int* start, const int* particles, const double* ref) {
    API_BEGIN(ctx)
    require(ctx->finalized, "update_rmsd before finalize");
    require(nforces == (int) ctx->rmsd.group.size(), "update_rmsd: the number of RMSD forces has changed");
    const size_t before = ctx->rmsd.atoms.size();
    CUDA_CHECK(cudaStreamSynchronize(ctx->stream));
    read_rmsd(ctx, "update_rmsd", nforces, start, particles, ref);
    upload_rmsd(ctx);
    ctx->rmd.atoms = ctx->rmsd.atomsDev.p; ctx->rmd.entryObj = ctx->rmsd.entryObjDev.p; ctx->rmd.ref = ctx->rmsd.refDev.p;
    ctx->rmd.nentries = (int) ctx->rmsd.atoms.size();
    // the same number of entries keeps the buffers and the launch shapes, so a captured step graph stays valid
    if (ctx->rmsd.atoms.size() != before) invalidate_graph(ctx);
    API_END(ctx)
}
static void setup_rmsd(b200md_ctx* c) {
    auto& r = c->rmsd;
    c->rmd = RmsdDev{};
    if (r.group.empty()) return;
    require(c->world == 1, "RMSDForce is not supported in multi-GPU runs");
    upload_rmsd(c);
    r.groupDev.upload(r.group);
    const size_t n = r.group.size();
    r.sums.alloc(16*n); r.sums.zero(); r.solved.alloc(16*n); r.solved.zero();
    RmsdDev& d = c->rmd;
    d.nobj = (int) n; d.nentries = (int) r.atoms.size();
    d.objStart = r.startDev.p; d.atoms = r.atomsDev.p; d.entryObj = r.entryObjDev.p; d.ref = r.refDev.p; d.refSq = r.refSqDev.p;
    d.group = r.groupDev.p; d.sums = r.sums.p; d.solved = r.solved.p;
    d.groupMask = 0xffffffffu;
}

// ---------------------------------------------------------------- CustomCVForce
extern "C" int b200md_set_cv_forces(b200md_ctx* ctx, int n) {
    API_BEGIN(ctx)
    check_set(ctx, "set_cv_forces", n);
    require(ctx->world == 1, "CustomCVForce is not supported in multi-GPU runs");
    ctx->cv.n = n;
    API_END(ctx)
}
static void setup_cv(b200md_ctx* c) {
    auto& v = c->cv;
    c->cvd = CvDev{};
    if (!v.n) return;
    require(c->world == 1, "CustomCVForce is not supported in multi-GPU runs");
    v.forces.alloc((size_t) v.n*3*c->npad); v.forces.zero();
    v.coeff.alloc(v.n); v.coeff.zero(); v.hcoeff.assign(v.n, 0.0);
    c->cvd.n = v.n; c->cvd.forces = v.forces.p; c->cvd.coeff = v.coeff.p;
    if (!c->evCv) CUDA_CHECK(cudaEventCreateWithFlags(&c->evCv, cudaEventDisableTiming));
}
static b200md_ctx* cv_pair(b200md_ctx* a, b200md_ctx* b, const char* call) {
    require(a && b && a != b, (std::string(call) + ": two different contexts are needed").c_str());
    require(a->finalized && b->finalized, (std::string(call) + " before finalize").c_str());
    require(a->device == b->device, (std::string(call) + ": the two contexts are on different devices").c_str());
    require(a->natoms == b->natoms && a->npad == b->npad, (std::string(call) + ": the two contexts differ in their number of particles").c_str());
    require(a->world == 1 && b->world == 1, (std::string(call) + ": not supported in multi-GPU runs").c_str());
    for (b200md_ctx* c : {a, b})
        if (!c->evCv) CUDA_CHECK(cudaEventCreateWithFlags(&c->evCv, cudaEventDisableTiming));
    return a;
}
extern "C" int b200md_cv_copy_state(b200md_ctx* from, b200md_ctx* to) {
    API_BEGIN(from)
    {
        cv_pair(from, to, "cv_copy_state");
        sync_positions(from);
        // stream-ordered on `from`'s stream, behind whatever `to` still has queued; `to` waits for the copy
        CUDA_CHECK(cudaEventRecord(to->evCv, to->stream));
        CUDA_CHECK(cudaStreamWaitEvent(from->stream, to->evCv, 0));
        launch_cv_copy_state(from->nb, to->nb, from->natoms, from->stream);
        from->kernelLaunches++;
        CUDA_CHECK(cudaEventRecord(from->evCv, from->stream));
        CUDA_CHECK(cudaStreamWaitEvent(to->stream, from->evCv, 0));
        if (from->haveBox) {
            bool same = to->haveBox;
            for (int i = 0; i < 3; i++) same = same && to->boxA[i] == from->boxA[i] && to->boxB[i] == from->boxB[i] && to->boxC[i] == from->boxC[i];
            if (!same) {
                for (int i = 0; i < 3; i++) { to->boxA[i] = from->boxA[i]; to->boxB[i] = from->boxB[i]; to->boxC[i] = from->boxC[i]; }
                to->haveBox = true;
                apply_box(to);
            }
        }
        // what b200md_set_positions does besides the upload
        to->stepStateValid = false;
        host_set_state(to);
        request_rebuild(to);
    }
    API_END(from)
}
extern "C" int b200md_cv_snapshot_forces(b200md_ctx* inner, b200md_ctx* outer, int slot) {
    API_BEGIN(outer)
    cv_pair(inner, outer, "cv_snapshot_forces");
    require(slot >= 0 && slot < outer->cv.n, "cv_snapshot_forces: slot out of range");
    const size_t n = 3*(size_t) outer->npad;
    // on the inner stream, behind the evaluation that produced the forces and before the next one; the outer stream waits
    CUDA_CHECK(cudaMemcpyAsync(outer->cv.forces.p + slot*n, inner->force.p, sizeof(long long)*n, cudaMemcpyDeviceToDevice, inner->stream));
    CUDA_CHECK(cudaEventRecord(inner->evCv, inner->stream));
    CUDA_CHECK(cudaStreamWaitEvent(outer->stream, inner->evCv, 0));
    API_END(outer)
}
extern "C" int b200md_set_cv_coefficients(b200md_ctx* ctx, int n, const double* d) {
    API_BEGIN(ctx)
    require(ctx->finalized, "set_cv_coefficients before finalize");
    require(n == ctx->cv.n, "set_cv_coefficients: n must be the number of collective variables");
    for (int i = 0; i < n; i++) require(std::isfinite(d[i]), "set_cv_coefficients: a coefficient is not finite");
    ctx->cv.hcoeff.assign(d, d + n);
    // stream ordered, into the buffer the step graphs read: no graph is captured or instantiated again
    if (n) CUDA_CHECK(cudaMemcpyAsync(ctx->cv.coeff.p, ctx->cv.hcoeff.data(), sizeof(double)*n, cudaMemcpyHostToDevice, ctx->stream));
    API_END(ctx)
}

// ---------------------------------------------------------------- state
// Multi-GPU (peer-memory data plane): only the owner integrates an atom.  Positions reach every rank with the step itself;
// velocities stay with the owner until somebody reads them from the host side.
static void sync_positions(b200md_ctx* c) { if (c->mg == MG_P2P && c->finalized) launch_pos_wait(c->nb, c->cd, c->stream); }
static void sync_velocities(b200md_ctx* c) {
    if (c->mg != MG_P2P || !c->velStale) return;
    launch_vel_push(c->nb, c->cd, c->stream);
    c->kernelLaunches += 2;
    c->velStale = false;
}
static void host_set_state(b200md_ctx* c) {       // the host wrote the full state on every rank: nothing to wait for
    if (c->mg != MG_P2P) return;
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
    // the blob's posq.w holds the charges of when it was saved; every other copy of the parameters is the context's own
    // (a checkpoint carries no force-field parameters, ContextImpl::loadCheckpoint)
    stamp_charges(ctx);
    CUDA_CHECK(cudaMemcpy(ctx->stepCounter.p, &h.rngStep, sizeof(unsigned long long), cudaMemcpyHostToDevice));
    host_set_state(ctx); ctx->velStale = false;
    if (ctx->haveBox) apply_box(ctx);
    request_rebuild(ctx);
    API_END(ctx)
}

// NCCL role split (replicated atoms): the LAST rank computes reciprocal space for all atoms and nothing else, so it keeps no
// neighbour list; the other world-1 ranks share the direct-space tiles (by i-block: list construction AND tile kernel) and
// the bonded terms
static bool nccl_pme_rank(const b200md_ctx* c) { return c->mg == MG_NCCL_SPLIT && c->rank == c->world - 1; }

// ---------------------------------------------------------------- force evaluation
// PME parameters of the next spread launch: the brick path needs a list that covers every atom on this GPU
static PmeDev pme_for_launch(const b200md_ctx* c) {
    PmeDev p = c->pme;
    p.brickAtoms = (c->pmeBrick && c->mg == MG_SINGLE && !c->pmeOnly && c->listBuilt) ? c->brickAtoms : 0;
    p.brickPoints = c->brickPoints;
    return p;
}

// Enqueue one force evaluation on the stream (no host sync).  Returns the number of kernels launched.
static int enqueue_forces(b200md_ctx* c, int terms, bool energy, bool forcesAlreadyZero = false, bool inStep = false, unsigned int groupMask = 0xffffffffu) {
    cudaStream_t s = c->stream;
    // ---- what this evaluation runs ----
    // NCCL role split: the PME rank does reciprocal space only, the direct ranks everything else.  The two halves of the
    // force field thus overlap on different GPUs, there is no charge-grid collective, and one int64 all-reduce of the force
    // buffer per step joins them.  NCCL without PME has no reciprocal space: every rank takes a share of everything.
    const bool p2p = c->mg == MG_P2P, nccl = c->mg == MG_NCCL_SPLIT || c->mg == MG_NCCL_SHARED;
    const bool pmeRank = nccl_pme_rank(c), directRank = c->mg == MG_NCCL_SPLIT && !pmeRank;
    const bool direct = (terms & B200MD_TERM_NB_DIRECT) && c->haveNb && !pmeRank;
    const bool recip = (terms & B200MD_TERM_NB_RECIP) && c->haveNb && c->nb.method == B200MD_NB_PME && !directRank;
    const int customBits = B200MD_TERM_CUSTOM_TORSIONS | B200MD_TERM_CUSTOM_BONDS | B200MD_TERM_CUSTOM_EXTERNALS | B200MD_TERM_CUSTOM_ANGLES |
                           B200MD_TERM_CUSTOM_COMPOUND | B200MD_TERM_CUSTOM_CENTROID;
    int bterms = terms & (B200MD_TERM_BONDS | B200MD_TERM_ANGLES | B200MD_TERM_TORSIONS | B200MD_TERM_RB_TORSIONS | B200MD_TERM_CMAP |
                          customBits);
    if (c->haveNb) bterms |= terms & B200MD_TERM_NB_DIRECT;
    const int nbonded = c->bd.nbonds + c->bd.nangles + c->bd.ntorsions + c->bd.nrb + c->bd.ncmap + c->bd.nexc;
    // the k_bonded branch is counted as one launch whenever it is taken (even when the selected classes have no terms and
    // launch_bonded skips the kernel); k_custom is counted once when it runs, for any number of custom classes, k_compound
    // once when it runs, the three centroid kernels when they run
    const bool classic = (bterms & ~customBits) && nbonded > 0;
    const bool custom = (bterms & c->ctd.terms) != 0;
    const bool compound = (bterms & B200MD_TERM_CUSTOM_COMPOUND) && c->cpd.nslots > 0;
    const bool centroid = (bterms & B200MD_TERM_CUSTOM_CENTROID) && c->ccd.nslots > 0;
    const bool rmsd = (terms & B200MD_TERM_RMSD) && c->rmd.nobj > 0;
    const bool bonded = (classic || custom || compound || centroid || rmsd) && !pmeRank;
    const bool cvForces = (terms & B200MD_TERM_CV_FORCES) && c->cvd.n > 0;
    // Reciprocal space (spread -> FFT/convolution -> gather, in USER atom order: independent of the neighbour list) and
    // direct space (list check / rebuild, tile kernel, bonded terms) are independent until the integrator: fork them onto
    // two streams (also inside the captured step graph).  Both accumulate into the same fixed-point force buffer, so the
    // overlap cannot change the result.  Never under NCCL, whose collectives of one communicator stay on one stream: there a
    // rank runs at most one of the two halves.
    const bool fork = direct && recip && c->overlapPme;
    cudaStream_t sp = fork ? c->streamPme : s;
    // The brick path of the spread walks the current list's sorted order, so when it runs beside direct space the
    // fork comes after the list build: the list then cannot flip under it (a rebuild flips at the end of k_build_tiles).
    // On one stream it runs before the build and reads the current list, which is complete even when stale.
    const PmeDev pme = pme_for_launch(c);
    const bool forkAfterList = fork && pme.brickAtoms > 0;
    // The bonded terms need nothing from the tile kernel either: on one GPU they fork with the spread onto a stream of their
    // own (not before the list build, whose wrap phase moves molecules in posq) and join before the integrator.
    const bool forkBonded = forkAfterList && bonded;
    // p2p: partial forces of the atoms this rank does not own -> the owners' inboxes.  Reciprocal space only ever touches the
    // atoms this rank OWNS (k_pme_gather), so when it runs on its own stream the push does not have to wait for it: it goes
    // out right behind the tile kernel and the bonded terms, beside the FFT chain.
    const bool pushEarly = p2p && fork;
    // Generalized Born: its pair passes walk this evaluation's list, so the chain forks after the list check and build (which
    // it needs even when direct space is not evaluated, e.g. GB alone in a force group) and joins before the integrator.  It
    // adds into the user-order fixed-point buffer like everything else, so the overlap cannot change the result.
    const bool gb = (terms & B200MD_TERM_GBSA) && c->gbsa.have && !pmeRank;
    const bool forkGb = gb && c->overlapPme;
    // CustomNonbondedForce: one pair kernel over this evaluation's list, forked and joined as the generalized Born chain is
    const bool cnb = (terms & B200MD_TERM_CUSTOM_NONBONDED) && c->cnb.have && !pmeRank;
    const bool forkCnb = cnb && c->overlapPme;
    CnbDev cnd = c->cnd; cnd.groupMask = groupMask;

    int launches = 0;
    auto launch_recip = [&]() {
        if (fork) {
            CUDA_CHECK(cudaEventRecord(c->evFork, s));
            CUDA_CHECK(cudaStreamWaitEvent(sp, c->evFork, 0));
        }
        if (recip) {
            launch_pme_spread(c->nb, pme, c->cd, sp, !forkAfterList); launches++;
            if (p2p) { launch_grid_push(c->pme, c->cd, sp); launches++; }
            launch_pme_fft_conv(c->nb, c->pme, c->cd, energy, fft_beside_tiles(c), sp); launches += pme_fft_launch_count(c->pme);
            launch_pme_gather(c->nb, pme, c->cd, sp); launches++;
        }
        if (fork) CUDA_CHECK(cudaEventRecord(c->evJoin, sp));
    };
    auto launch_bonded_terms = [&](cudaStream_t sb) {
        BondedDev bd = c->bd; bd.groupMask = groupMask;
        CustomDev ct = c->ctd; ct.groupMask = groupMask;
        CompoundDev cp = c->cpd; cp.groupMask = groupMask;
        CompoundDev cc = c->ccd; cc.groupMask = groupMask;
        launch_bonded(c->nb, bd, ct, cp, cc, c->cen, bterms, energy, sb);
        launches += (classic ? 1 : 0) + (custom ? 1 : 0) + (compound ? 1 : 0) + (centroid ? CENTROID_LAUNCHES : 0);
        if (rmsd) {
            RmsdDev rd = c->rmd; rd.groupMask = groupMask;
            launch_rmsd(c->nb, rd, energy, sb);
            launches += RMSD_LAUNCHES;
        }
    };

    // ---- the schedule, in stream order ----
    if (!forcesAlreadyZero) CUDA_CHECK(cudaMemsetAsync(c->force.p, 0, sizeof(long long)*3*c->npad, s));
    if (energy) CUDA_CHECK(cudaMemsetAsync(c->energy.p, 0, sizeof(double)*B200MD_NUM_ENERGY, s));
    if (p2p && !direct) { launch_pos_wait(c->nb, c->cd, s); launches++; }       // nobody else on this stream waits for the owners' position stores
    if (cvForces) { launch_cv_combine(c->nb, c->cvd, s); launches++; }
    if (!forkAfterList) launch_recip();
    else {
        // the charge grid is zeroed at the head of the step on the chain's stream, beside the list check and build: it needs
        // nothing from them, and as the spread's first node it sat on the chain, which is the step's longest path (DHFR:
        // memset 1.6 us plus a node gap before the spread)
        CUDA_CHECK(cudaEventRecord(c->evForkGrid, s));
        CUDA_CHECK(cudaStreamWaitEvent(sp, c->evForkGrid, 0));
        CUDA_CHECK(cudaMemsetAsync(pme.gridFixed, 0, sizeof(long long)*(size_t) pme.nx*pme.ny*pme.nz, sp));
    }
    if (direct || gb || cnb) {
        launch_check_displacement(c->nb, c->cd, s); launches++;
        launch_list_build(c->nb, s); launches += LIST_BUILD_LAUNCHES;
    }
    if (forkGb) {
        CUDA_CHECK(cudaEventRecord(c->gbsa.evFork, s));
        CUDA_CHECK(cudaStreamWaitEvent(c->gbsa.stream, c->gbsa.evFork, 0));
        launch_gbsa(c->nb, c->gbd, energy, c->gbsa.stream);
        CUDA_CHECK(cudaEventRecord(c->gbsa.evJoin, c->gbsa.stream));
    }
    if (gb) launches += GBSA_LAUNCHES;
    if (forkCnb) {
        CUDA_CHECK(cudaEventRecord(c->cnb.evFork, s));
        CUDA_CHECK(cudaStreamWaitEvent(c->cnb.stream, c->cnb.evFork, 0));
        launch_custom_nonbonded(c->nb, cnd, energy, c->cnb.stream);
        CUDA_CHECK(cudaEventRecord(c->cnb.evJoin, c->cnb.stream));
    }
    if (cnb) launches++;
    if (forkAfterList) launch_recip();
    if (forkBonded) {
        CUDA_CHECK(cudaStreamWaitEvent(c->streamBonded, c->evFork, 0));
        launch_bonded_terms(c->streamBonded);
        CUDA_CHECK(cudaEventRecord(c->evJoinBonded, c->streamBonded));
    }
    if (direct) { launch_pair(c->nb, energy, s); launches += PAIR_LAUNCHES; }
    if (bonded && !forkBonded) launch_bonded_terms(s);
    if (gb && !forkGb) launch_gbsa(c->nb, c->gbd, energy, s);
    if (cnb && !forkCnb) launch_custom_nonbonded(c->nb, cnd, energy, s);
    if (pushEarly) { launch_force_push(c->nb, c->cd, s); launches++; }
    if (fork) CUDA_CHECK(cudaStreamWaitEvent(s, c->evJoin, 0));
    if (forkBonded) CUDA_CHECK(cudaStreamWaitEvent(s, c->evJoinBonded, 0));
    if (forkGb) CUDA_CHECK(cudaStreamWaitEvent(s, c->gbsa.evJoin, 0));
    if (forkCnb) CUDA_CHECK(cudaStreamWaitEvent(s, c->cnb.evJoin, 0));
    if (p2p) {
        if (!pushEarly) { launch_force_push(c->nb, c->cd, s); launches++; }
        // in the step path k_integrate totals own partial + inboxes; here (energies, getState) the owners total and broadcast
        // so that every rank ends up with every force
        if (!inStep) { launch_force_total(c->nb, c->cd, s); launches += 2; }
    }
    if (nccl && g_nccl.AllReduce(c->force.p, c->force.p, (size_t) 3*c->npad, NCCL_INT64, NCCL_SUM, c->comm, s) != 0)
        throw std::runtime_error("ncclAllReduce(force) failed");
    // the energies are summed over the ranks in every multi-GPU mode, p2p included
    if (c->mg != MG_SINGLE && energy && g_nccl.AllReduce(c->energy.p, c->energy.p, B200MD_NUM_ENERGY, NCCL_FLOAT64, NCCL_SUM, c->comm, s) != 0)
        throw std::runtime_error("ncclAllReduce(energy) failed");
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
    if (!c->listDirty || !(c->haveNb || c->gbsa.have || c->cnb.have)) { c->listDirty = false; return; }
    if (c->pmeOnly || nccl_pme_rank(c)) { c->listDirty = false; return; }    // keeps no list
    for (int attempt = 0; attempt < 8; attempt++) {
        launch_check_displacement(c->nb, c->cd, c->stream);
        launch_list_build(c->nb, c->stream);
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
        if (terms & (B200MD_TERM_CUSTOM_TORSIONS | B200MD_TERM_CUSTOM_BONDS | B200MD_TERM_CUSTOM_EXTERNALS | B200MD_TERM_CUSTOM_ANGLES |
                     B200MD_TERM_CUSTOM_COMPOUND | B200MD_TERM_CUSTOM_CENTROID)) e += h[EN_CUSTOM];
        if ((terms & B200MD_TERM_GBSA) && ctx->gbsa.have) e += h[EN_GB];
        if (terms & B200MD_TERM_RMSD) e += h[EN_RMSD];
        if ((terms & B200MD_TERM_CUSTOM_NONBONDED) && ctx->cnb.have) {
            e += h[EN_CNB];
            for (int o = 0; o < ctx->cnb.nobj; o++)        // ReferenceCalcCustomNonbondedForceKernel::execute
                if ((bonded_group_mask >> ctx->cnb.group[o]) & 1u) e += ctx->cnb.lrc[o]/ctx->nb.box.volume;
        }
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
    ctx->velStale = ctx->mg == MG_P2P;
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
    const cudaError_t e = cudaGraphInstantiate(exec, g, c->mg == MG_SINGLE ? cudaGraphInstantiateFlagUseNodePriority : 0);
    cudaGraphDestroy(g);
    CUDA_CHECK(e);
    c->graphInstantiations++;
}

extern "C" int b200md_step(b200md_ctx* ctx, int nsteps) {
    API_BEGIN(ctx)
    require(ctx->finalized && ctx->haveIntegrator, "step before finalize / set_integrator");
    // the coefficients of the collective-variable forces come from the host before every step
    require(ctx->cv.n == 0 || nsteps <= 1, "step: a context with CustomCVForce terms takes one step per call");
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
        c->velStale = c->mg == MG_P2P;
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

extern "C" int b200md_get_list(b200md_ctx* ctx, int* sorig, int64_t cap, int* tile_i, int* tile_j, unsigned int* tile_mask, int64_t* ntiles) {
    API_BEGIN(ctx)
    require(ctx->finalized, "get_list before finalize");
    const DevFlags f = read_flags(ctx, true);
    const ListBufs& L = ctx->lists[f.ct[CT_CUR] & 1];
    const int pool = ctx->nb.maxTiles/TILE_REGIONS;
    int64_t total = 0;
    for (int r = 0; r < TILE_REGIONS; r++) total += std::min(f.cur()[LC_TILES + r], pool);
    *ntiles = total;
    if (sorig) CUDA_CHECK(cudaMemcpy(sorig, L.sorig.p, sizeof(int)*ctx->npad, cudaMemcpyDeviceToHost));
    if (tile_i && tile_j && tile_mask) {
        require(cap >= total, "get_list: the tile arrays are smaller than the list");
        std::vector<int> ti(ctx->nb.maxTiles), tj((size_t) ctx->nb.maxTiles*32), tm(ctx->nb.maxTiles);
        std::vector<unsigned int> mp((size_t) ctx->nb.maxTiles*32);
        CUDA_CHECK(cudaMemcpy(ti.data(), L.tileI.p, sizeof(int)*ti.size(), cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(tj.data(), L.tileJ.p, sizeof(int)*tj.size(), cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(tm.data(), L.tileMask.p, sizeof(int)*tm.size(), cudaMemcpyDeviceToHost));
        CUDA_CHECK(cudaMemcpy(mp.data(), L.maskPool.p, sizeof(unsigned int)*mp.size(), cudaMemcpyDeviceToHost));
        int64_t o = 0;
        for (int r = 0; r < TILE_REGIONS; r++)
            for (int k = 0; k < std::min(f.cur()[LC_TILES + r], pool); k++, o++) {
                const size_t t = (size_t) r*pool + k;
                tile_i[o] = ti[t];
                for (int l = 0; l < 32; l++) {
                    tile_j[o*32 + l] = tj[t*32 + l];
                    tile_mask[o*32 + l] = tm[t] < 0 ? 0xffffffffu : mp[(size_t) tm[t]*32 + l];
                }
            }
    }
    API_END(ctx)
}

extern "C" int b200md_time_phase(b200md_ctx* ctx, int phase, int reps, double* ms_mean) {
    API_BEGIN(ctx)
    require(ctx->finalized, "time_phase before finalize");
    b200md_ctx* c = ctx;
    prepare_list(c);
    c->stepStateValid = false;            // phases 0, 3, 6 accumulate into the force buffer, phase 5 flips the list
    cudaStream_t s = c->stream;
    CommDev local{}; local.world = 1;   // phases are timed rank-locally (no peer traffic, no waits)
    cudaEvent_t e0, e1;
    CUDA_CHECK(cudaEventCreate(&e0)); CUDA_CHECK(cudaEventCreate(&e1));
    double total = 0;
    // the integrate phase mutates the state: positions and velocities are restored before every repetition, the step
    // counter (which each repetition advances, as a step does) once at the end
    Snapshot state, counter;
    require(phase != 7 || c->ctd.nslots > 0, "time_phase(custom torsions): the System has none");
    require(phase != 8 || c->cpd.nslots > 0, "time_phase(custom compound bonds): the System has none");
    require(phase != 9 || c->ccd.nslots > 0, "time_phase(custom centroid bonds): the System has none");
    require(phase != 10 || c->gbsa.have, "time_phase(generalized Born): the System has none");
    require(phase != 13 || c->rmd.nobj > 0, "time_phase(RMSD): the System has none");
    require(phase != 14 || c->cnb.have, "time_phase(custom nonbonded): the System has none");
    if (phase == 4) {
        require(c->haveIntegrator, "time_phase(integrate) before set_integrator");
        state.parts = state_spans(c, ST_POS | ST_VEL); state.save(s);
        counter.parts = {{c->stepCounter.p, sizeof(unsigned long long)}}; counter.save(s);
    }
    for (int r = -2; r < reps; r++) {
        if (phase == 4) state.restore(s);
        if (phase == 5 || phase == 11 || phase == 12) set_counter(c, CT_REBUILD, 1);     // the list is not marked dirty: the next step adds no synchronous rebuild
        if (phase == 0) { CUDA_CHECK(cudaMemsetAsync(&c->counters.p[CT_CURSOR], 0, sizeof(int), s)); CUDA_CHECK(cudaMemsetAsync(&c->counters.p[CT_PAIRSTART], 0, sizeof(int), s)); }      // the SM-partitioned tile kernel's cursor starts from tile 0
        if (phase == 12) launch_list_prep(c->nb, s);        // untimed: the tile pass reads what the prep pass sorted
        CUDA_CHECK(cudaEventRecord(e0, s));
        switch (phase) {
            case 0: launch_pair(c->nb, false, s); break;
            case 1: launch_pme_spread(c->nb, pme_for_launch(c), local, s); break;
            case 2: launch_pme_fft_conv(c->nb, c->pme, local, false, fft_beside_tiles(c), s); break;
            case 3: launch_pme_gather(c->nb, pme_for_launch(c), local, s); break;
            case 4: launch_integrate(c->nb, c->units, c->integ, local, s); break;
            case 5: launch_list_build(c->nb, s); break;
            case 6: launch_bonded(c->nb, c->bd, c->ctd, c->cpd, c->ccd, c->cen, B200MD_TERM_ALL, false, s); break;
            case 7: launch_custom(c->nb, c->ctd, B200MD_TERM_ALL, false, s); break;
            case 8: launch_compound(c->nb, c->cpd, false, s); break;
            case 9: launch_centroid(c->nb, c->ccd, c->cen, false, s); break;
            case 10: launch_gbsa(c->nb, c->gbd, false, s); break;
            case 11: launch_list_prep(c->nb, s); break;
            case 12: launch_build_tiles(c->nb, s); break;
            case 13: launch_rmsd(c->nb, c->rmd, false, s); break;
            case 14: launch_custom_nonbonded(c->nb, c->cnd, false, s); break;
            default: throw std::runtime_error("unknown phase");
        }
        CUDA_CHECK(cudaEventRecord(e1, s));
        if (phase == 11) launch_build_tiles(c->nb, s);      // untimed: completes the build (and flips the list) as phase 5 does
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
