// B200Platform.cpp -- libOpenMMB200.so: the OpenMM Platform plugin for the CUDA-native (sm_90a) hot path.
//
// A thin C++ adapter: every KernelImpl below forwards one abstract kernel interface of the reference
// (olla/include/openmm/kernels.h) to the C-ABI of libb200md.so (include/b200md.h), where all the CUDA lives.
// Loaded by Platform::loadPluginLibrary / loadPluginsFromDirectory (olla/src/Platform.cpp:221-320) through the
// extern "C" registerPlatforms() entry point (PluginInitializer.h:47), exactly like platforms/cuda
// (CudaPlatform.cpp:59-61).  Compiled against the reference's headers where they lie; no reference source is copied.
//
// Supported: NonbondedForce (NoCutoff, CutoffNonPeriodic, CutoffPeriodic, PME; parameter offsets), HarmonicBondForce,
// HarmonicAngleForce, PeriodicTorsionForce, RBTorsionForce, CMAPTorsionForce, CustomTorsionForce (any number of objects, each
// in its own force group; custom torsions without energy parameter derivatives, expressions within the limits of
// custom_translate.h), CMMotionRemover;
// Verlet / Langevin / LangevinMiddle integrators; SETTLE + X-H_n SHAKE constraints; MonteCarloBarostat and
// MonteCarloAnisotropicBarostat (ApplyMonteCarloBarostatKernel; MonteCarloMembraneBarostat is refused).  A Force class without a kernel here
// makes Platform::supportsKernels() false; an unsupported OPTION of a supported class is rejected in contextCreated()
// (validateSystem), which is the only place from which ContextImpl falls back to the next platform (ContextImpl.cpp:152-166).
//
// Bonded classes.  Each keeps the terms of all its Force objects in one TermRecord of PlatformData, sent at finalize; what
// their kernels share (ObjectTerms: the object's range of the record, group tags, updates) exists once.  Bond, angle,
// periodic-torsion and RB-torsion kernels are one template, B200CalcBondedForceKernel; CMAP and custom torsions keep
// their own kernels for their maps and expression programs.
//
// The hot loop.  Integrator::step(n) of the reference is, per step, updateContextState() -> calcForcesAndEnergy(true,
// false, groups) -> Integrate*StepKernel::execute (LangevinIntegrator.cpp:74-82).  Here a forces-only evaluation is
// LAZY: finishComputation records what was asked for and returns; when the integrator kernel's execute() follows and the
// request covered the whole force field, ONE b200md_step(1) replays the captured step graph (list check, tile kernel,
// reciprocal space, bonded terms, fused integrate + constraints + CM removal).  Anything that needs the forces before
// that (getForces, kinetic energy, energies) flushes the pending evaluation with b200md_compute first.
#include "openmm/Platform.h"
#include "openmm/KernelFactory.h"
#include "openmm/kernels.h"
#include "openmm/OpenMMException.h"
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/NonbondedForce.h"
#include "openmm/HarmonicBondForce.h"
#include "openmm/HarmonicAngleForce.h"
#include "openmm/PeriodicTorsionForce.h"
#include "openmm/RBTorsionForce.h"
#include "openmm/CMAPTorsionForce.h"
#include "openmm/CustomTorsionForce.h"
#include "openmm/CMMotionRemover.h"
#include "openmm/VerletIntegrator.h"
#include "openmm/LangevinIntegrator.h"
#include "openmm/LangevinMiddleIntegrator.h"
#include "openmm/MonteCarloMembraneBarostat.h"
#include "openmm/internal/ContextImpl.h"
#include "openmm/internal/NonbondedForceImpl.h"
#include "openmm/internal/CMAPTorsionForceImpl.h"
#include "../include/b200md.h"
#include "custom_translate.h"
#include <algorithm>
#include <map>
#include <string>
#include <vector>
#include <sstream>
#include <cstdlib>

using namespace OpenMM;
using namespace std;

namespace {

// next grid size whose prime factors are <= 13 (what the bespoke FFT handles; the reference CUDA platform rounds to
// 2,3,5,7-smooth sizes the same way, CudaKernels.cpp:698-700)
int fftFriendly(int n) {
    for (;; n++) {
        int r = n;
        for (int p : {2, 3, 5, 7, 11, 13}) while (r % p == 0) r /= p;
        if (r == 1) return n;
    }
}

// The terms of one bonded class over all its Force objects, as the arrays its b200md_set_* call takes: one column per
// array, each holding the same number of entries for every term (bonds: atoms p1, p2 and parameters length, k; CMAP: one
// atom column of 8 per term).  ints are the integer parameters: torsion periodicity, CMAP map, custom-torsion program.
struct TermRecord {
    int kind;                       // B200MD_BONDED_*
    vector<vector<int> > atoms, ints;
    vector<vector<double> > params;
    vector<int> group;              // the force group of the term's Force, | 0x80 if it uses periodic boundary conditions
    TermRecord(int kind, int numAtoms, int numInts, int numParams) : kind(kind), atoms(numAtoms), ints(numInts), params(numParams) {}
    int size() const { return (int) group.size(); }
    // appends one term, each list split evenly over its columns
    void add(const vector<int>& a, const vector<int>& n, const vector<double>& p) { split(a, atoms); split(n, ints); split(p, params); }
    template<class T> static void split(const vector<T>& v, vector<vector<T> >& columns) {
        const size_t w = columns.empty() ? 0 : v.size()/columns.size();
        for (size_t c = 0; c < columns.size(); c++) columns[c].insert(columns[c].end(), v.begin() + c*w, v.begin() + (c+1)*w);
    }
};

// What the bond, angle, periodic-torsion and RB-torsion kernels differ in (B200CalcBondedForceKernel below): the Force,
// the term bit, the names in messages, how term i is read into the record, and the calls that send the record.
struct Bonds {
    typedef HarmonicBondForce Force; typedef CalcHarmonicBondForceKernel Kernel;
    enum { bit = B200MD_TERM_BONDS };
    static constexpr const char* name = "HarmonicBondForce", *terms = "bonds", *aTerm = "a bond";
    static int count(const Force& f) { return f.getNumBonds(); }
    static void read(const Force& f, int i, TermRecord& r) { int a, b; double r0, k; f.getBondParameters(i, a, b, r0, k); r.add({a, b}, {}, {r0, k}); }
    static int set(b200md_ctx* c, const TermRecord& r) { return b200md_set_bonds(c, r.size(), r.atoms[0].data(), r.atoms[1].data(), r.params[0].data(), r.params[1].data()); }
    static int update(b200md_ctx* c, const TermRecord& r) { return b200md_update_bonded_params(c, r.kind, r.size(), r.params[0].data(), r.params[1].data(), nullptr); }
};
struct Angles {
    typedef HarmonicAngleForce Force; typedef CalcHarmonicAngleForceKernel Kernel;
    enum { bit = B200MD_TERM_ANGLES };
    static constexpr const char* name = "HarmonicAngleForce", *terms = "angles", *aTerm = "an angle";
    static int count(const Force& f) { return f.getNumAngles(); }
    static void read(const Force& f, int i, TermRecord& r) { int a, b, c; double t0, k; f.getAngleParameters(i, a, b, c, t0, k); r.add({a, b, c}, {}, {t0, k}); }
    static int set(b200md_ctx* c, const TermRecord& r) {
        return b200md_set_angles(c, r.size(), r.atoms[0].data(), r.atoms[1].data(), r.atoms[2].data(), r.params[0].data(), r.params[1].data());
    }
    static int update(b200md_ctx* c, const TermRecord& r) { return b200md_update_bonded_params(c, r.kind, r.size(), r.params[0].data(), r.params[1].data(), nullptr); }
};
struct Torsions {
    typedef PeriodicTorsionForce Force; typedef CalcPeriodicTorsionForceKernel Kernel;
    enum { bit = B200MD_TERM_TORSIONS };
    static constexpr const char* name = "PeriodicTorsionForce", *terms = "torsions", *aTerm = "a torsion";
    static int count(const Force& f) { return f.getNumTorsions(); }
    static void read(const Force& f, int i, TermRecord& r) { int a, b, c, e, n; double ph, k; f.getTorsionParameters(i, a, b, c, e, n, ph, k); r.add({a, b, c, e}, {n}, {ph, k}); }
    static int set(b200md_ctx* c, const TermRecord& r) {
        return b200md_set_torsions(c, r.size(), r.atoms[0].data(), r.atoms[1].data(), r.atoms[2].data(), r.atoms[3].data(), r.ints[0].data(), r.params[0].data(), r.params[1].data());
    }
    static int update(b200md_ctx* c, const TermRecord& r) { return b200md_update_bonded_params(c, r.kind, r.size(), r.params[0].data(), r.params[1].data(), r.ints[0].data()); }
};
struct RBTorsions {
    typedef RBTorsionForce Force; typedef CalcRBTorsionForceKernel Kernel;
    enum { bit = B200MD_TERM_RB_TORSIONS };
    static constexpr const char* name = "RBTorsionForce", *terms = "torsions", *aTerm = "a torsion";
    static int count(const Force& f) { return f.getNumTorsions(); }
    static void read(const Force& f, int i, TermRecord& r) {
        int a, b, c, e; double c0, c1, c2, c3, c4, c5;
        f.getTorsionParameters(i, a, b, c, e, c0, c1, c2, c3, c4, c5);
        r.add({a, b, c, e}, {}, {c0, c1, c2, c3, c4, c5});
    }
    static int set(b200md_ctx* c, const TermRecord& r) { return b200md_set_rb_torsions(c, r.size(), r.atoms[0].data(), r.atoms[1].data(), r.atoms[2].data(), r.atoms[3].data(), r.params[0].data()); }
    static int update(b200md_ctx* c, const TermRecord& r) { return b200md_update_rb_torsion_params(c, r.size(), r.params[0].data()); }
};

// per-Context state (ContextImpl::setPlatformData)
struct PlatformData {
    b200md_ctx* ctx = nullptr;
    int numParticles = 0;
    bool finalized = false;
    int pendingTerms = 0;
    bool includeEnergy = false;
    // lazy forces-only evaluation (see the header comment)
    bool lazyForces = false;
    int lazyTerms = 0;
    unsigned int lazyGroups = 0;
    int systemTerms = 0;            // every term the System has a kernel for
    unsigned int bondedGroupsUsed = 0;
    int cmFrequency = 0;
    bool cmRequested = false;       // RemoveCMMotionKernel::execute seen since the last integrator step
    bool useFusedStep = true;       // B200MD_PLUGIN_FUSED=0: always compute + integrate_only (debugging)
    // the bonded terms of every Force object, one record per class (columns: atoms, integer parameters, parameters), sent at finalize
    TermRecord bonds{B200MD_BONDED_BONDS, 2, 0, 2}, angles{B200MD_BONDED_ANGLES, 3, 0, 2}, torsions{B200MD_BONDED_TORSIONS, 4, 1, 2},
               rb{B200MD_BONDED_RB_TORSIONS, 4, 0, 1}, cmap{B200MD_BONDED_CMAP, 1, 1, 0}, custom{B200MD_BONDED_CUSTOM_TORSIONS, 1, 1, 1};
    // CMAP: the maps of all objects one after the other (a term's map index counts from the first map of all objects);
    // coefficients from CMAPTorsionForceImpl::calcMapDerivatives, [sum size^2][16]
    vector<int> cmapSize; vector<double> cmapCoeff;
    // custom torsions: the programs of all objects one after the other (object f's expression is the pair 2f, 2f+1); the
    // parameters of every term padded to B200MD_CUSTOM_MAX_PARAMS in the record, packed to the widest object's count when sent
    vector<int> customProgStart = vector<int>(1, 0), customOp, customArg; vector<double> customImm;
    int customStride = 0;
    // the global parameters the expressions read: slot of every name (shared by all objects) and the value last sent
    map<string, int> customGlobalSlot;
    vector<double> customGlobals;
    vector<double> packedCustomParams() const {
        const size_t n = custom.size();
        vector<double> p(n*customStride);
        for (size_t i = 0; i < n; i++)
            for (int k = 0; k < customStride; k++) p[i*customStride + k] = custom.params[0][i*B200MD_CUSTOM_MAX_PARAMS + k];
        return p;
    }
    map<string, string> props;
    // a box b200md_set_box refused (smaller than twice the cutoff): the reference raises that at the next force evaluation
    // (ReferenceKernels.cpp:983-985), not in setPeriodicBoxVectors; a later box that passes clears it
    string boxError;
    int integratorKind = -1;
    double dt = 0, temperature = 0, friction = 0, tol = 0;
    int seed = 0;
    void check(int rc) const {
        if (rc != 0) throw OpenMMException(string("B200 platform: ") + b200md_last_error(ctx));
    }
    void checkBox() const {
        if (!boxError.empty()) throw OpenMMException(boxError);
    }
    void ensureFinalized() {
        if (finalized) return;
        if (bonds.size()) check(Bonds::set(ctx, bonds));
        if (angles.size()) check(Angles::set(ctx, angles));
        if (torsions.size()) check(Torsions::set(ctx, torsions));
        if (rb.size()) check(RBTorsions::set(ctx, rb));
        if (cmap.size()) check(b200md_set_cmap(ctx, (int) cmapSize.size(), cmapSize.data(), cmapCoeff.data(), cmap.size(), cmap.ints[0].data(), cmap.atoms[0].data()));
        for (const TermRecord* r : {&bonds, &angles, &torsions, &rb, &cmap})
            if (r->size()) check(b200md_set_bonded_groups(ctx, r->kind, r->size(), r->group.data()));
        if (custom.size()) {
            const vector<double> par = packedCustomParams();
            check(b200md_set_custom_torsions(ctx, (int) customProgStart.size()/2, customProgStart.data(), customOp.data(), customArg.data(),
                                             customImm.data(), customStride, custom.size(), custom.ints[0].data(), custom.atoms[0].data(), par.data()));
            check(b200md_set_bonded_groups(ctx, custom.kind, custom.size(), custom.group.data()));
        }
        if (!customGlobals.empty()) check(b200md_set_custom_globals(ctx, (int) customGlobals.size(), customGlobals.data()));
        check(b200md_finalize(ctx));
        finalized = true;
    }
    // a pending forces-only evaluation becomes real (someone reads the forces before an integrator step consumes it)
    void flushForces() {
        if (!lazyForces) return;
        lazyForces = false;
        check(b200md_compute_groups(ctx, lazyTerms, lazyGroups, 1, nullptr));
    }
    void dropForces() { lazyForces = false; }
    // RemoveCMMotionKernel::execute is deferred too: the fused step removes the centre-of-mass motion itself
    void flushCm() {
        if (!cmRequested) return;
        cmRequested = false;
        if (cmFrequency > 0 && b200md_get_step_count(ctx) % cmFrequency == 0) check(b200md_remove_cm_motion(ctx));
    }
};

PlatformData& getData(ContextImpl& context) { return *reinterpret_cast<PlatformData*>(context.getPlatformData()); }
const PlatformData& getData(const ContextImpl& context) { return *reinterpret_cast<const PlatformData*>(const_cast<ContextImpl&>(context).getPlatformData()); }

// ------------------------------------------------------------------------------------------------ mandatory kernels
class B200CalcForcesAndEnergyKernel : public CalcForcesAndEnergyKernel {
public:
    B200CalcForcesAndEnergyKernel(string name, const Platform& platform) : CalcForcesAndEnergyKernel(name, platform) {}
    void initialize(const System& system) {}
    void beginComputation(ContextImpl& context, bool includeForce, bool includeEnergy, int groups) {
        PlatformData& d = getData(context);
        d.checkBox();
        d.ensureFinalized();
        d.dropForces();             // superseded by this evaluation
        d.pendingTerms = 0;
        d.includeEnergy = includeEnergy;
    }
    double finishComputation(ContextImpl& context, bool includeForce, bool includeEnergy, int groups, bool& valid) {
        // every Calc*ForceKernel::execute only recorded its term; one engine call evaluates them all on the device
        PlatformData& d = getData(context);
        double energy = 0;
        valid = true;
        if (includeForce && !includeEnergy) {
            d.lazyForces = true; d.lazyTerms = d.pendingTerms; d.lazyGroups = (unsigned int) groups;
            return 0.0;
        }
        d.check(b200md_compute_groups(d.ctx, d.pendingTerms, (unsigned int) groups, includeForce ? 1 : 0, includeEnergy ? &energy : nullptr));
        return energy;
    }
};

class B200UpdateStateDataKernel : public UpdateStateDataKernel {
public:
    B200UpdateStateDataKernel(string name, const Platform& platform) : UpdateStateDataKernel(name, platform) {}
    void initialize(const System& system) {
        // masses and constraints belong to the System, not to a Force: hand them over here (once per Context)
        // (done in B200Platform::contextCreated, which has the ContextImpl)
    }
    double getTime(const ContextImpl& context) const { return b200md_get_time(getData(context).ctx); }
    void setTime(ContextImpl& context, double time) { b200md_set_time(getData(context).ctx, time); }
    void getPositions(ContextImpl& context, vector<Vec3>& positions) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        vector<double> x(3*d.numParticles);
        d.check(b200md_get_positions(d.ctx, x.data()));
        positions.resize(d.numParticles);
        for (int i = 0; i < d.numParticles; i++) positions[i] = Vec3(x[3*i], x[3*i+1], x[3*i+2]);
    }
    void setPositions(ContextImpl& context, const vector<Vec3>& positions) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        vector<double> x(3*d.numParticles);
        for (int i = 0; i < d.numParticles; i++) for (int k = 0; k < 3; k++) x[3*i+k] = positions[i][k];
        d.check(b200md_set_positions(d.ctx, x.data()));
    }
    void getVelocities(ContextImpl& context, vector<Vec3>& velocities) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.flushCm();
        vector<double> x(3*d.numParticles);
        d.check(b200md_get_velocities(d.ctx, x.data()));
        velocities.resize(d.numParticles);
        for (int i = 0; i < d.numParticles; i++) velocities[i] = Vec3(x[3*i], x[3*i+1], x[3*i+2]);
    }
    void setVelocities(ContextImpl& context, const vector<Vec3>& velocities) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.cmRequested = false;
        vector<double> x(3*d.numParticles);
        for (int i = 0; i < d.numParticles; i++) for (int k = 0; k < 3; k++) x[3*i+k] = velocities[i][k];
        d.check(b200md_set_velocities(d.ctx, x.data()));
    }
    void getForces(ContextImpl& context, vector<Vec3>& forces) {
        PlatformData& d = getData(context);
        d.checkBox();
        d.ensureFinalized();
        d.flushForces();
        vector<double> x(3*d.numParticles);
        d.check(b200md_get_forces(d.ctx, x.data()));
        forces.resize(d.numParticles);
        for (int i = 0; i < d.numParticles; i++) forces[i] = Vec3(x[3*i], x[3*i+1], x[3*i+2]);
    }
    void getEnergyParameterDerivatives(ContextImpl& context, map<string, double>& derivs) {}
    void getPeriodicBoxVectors(ContextImpl& context, Vec3& a, Vec3& b, Vec3& c) const {
        double x[3], y[3], z[3];
        b200md_get_box(getData(context).ctx, x, y, z);
        a = Vec3(x[0], x[1], x[2]); b = Vec3(y[0], y[1], y[2]); c = Vec3(z[0], z[1], z[2]);
    }
    void setPeriodicBoxVectors(ContextImpl& context, const Vec3& a, const Vec3& b, const Vec3& c) {
        PlatformData& d = getData(context);
        const double x[3] = {a[0], a[1], a[2]}, y[3] = {b[0], b[1], b[2]}, z[3] = {c[0], c[1], c[2]};
        d.dropForces();
        if (b200md_set_box(d.ctx, x, y, z) != 0) d.boxError = string("B200 platform: ") + b200md_last_error(d.ctx);
        else d.boxError.clear();
    }
    void createCheckpoint(ContextImpl& context, ostream& stream) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.flushCm();
        int64_t n = b200md_checkpoint_save(d.ctx, nullptr, 0);
        vector<char> buf(n);
        if (b200md_checkpoint_save(d.ctx, buf.data(), n) != n) d.check(-1);
        stream.write((const char*) &n, sizeof(n));
        stream.write(buf.data(), n);
    }
    void loadCheckpoint(ContextImpl& context, istream& stream) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces(); d.cmRequested = false;
        int64_t n = 0;
        stream.read((char*) &n, sizeof(n));
        // a blob of the other precision differs in size; b200md_checkpoint_load reads its header and names the mismatch
        const int64_t expect = b200md_checkpoint_save(d.ctx, nullptr, 0);
        if (n <= 0 || n > 2*expect) throw OpenMMException("B200 platform: checkpoint does not match this Context");
        vector<char> buf(n);
        stream.read(buf.data(), n);
        d.check(b200md_checkpoint_load(d.ctx, buf.data(), n));
        if (n != expect) throw OpenMMException("B200 platform: checkpoint does not match this Context");
    }
};

class B200ApplyConstraintsKernel : public ApplyConstraintsKernel {
public:
    B200ApplyConstraintsKernel(string name, const Platform& platform) : ApplyConstraintsKernel(name, platform) {}
    void initialize(const System& system) {}
    void apply(ContextImpl& context, double tol) { PlatformData& d = getData(context); d.ensureFinalized(); d.dropForces(); d.check(b200md_apply_constraints(d.ctx, tol)); }
    void applyToVelocities(ContextImpl& context, double tol) { PlatformData& d = getData(context); d.ensureFinalized(); d.flushCm(); d.check(b200md_apply_velocity_constraints(d.ctx, tol)); }
};

class B200VirtualSitesKernel : public VirtualSitesKernel {
public:
    B200VirtualSitesKernel(string name, const Platform& platform) : VirtualSitesKernel(name, platform) {}
    void initialize(const System& system) {
        for (int i = 0; i < system.getNumParticles(); i++)
            if (system.isVirtualSite(i)) throw OpenMMException("B200 platform: virtual sites are not supported");
    }
    void computePositions(ContextImpl& context) {}
};

// ------------------------------------------------------------------------------------------------ forces
class B200CalcNonbondedForceKernel : public CalcNonbondedForceKernel {
public:
    B200CalcNonbondedForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcNonbondedForceKernel(name, platform), context(context), alpha(0) {
        grid[0] = grid[1] = grid[2] = 0;
    }
    // base parameters + offsets (NonbondedForce::addParticleParameterOffset / addExceptionParameterOffset)
    struct Offset { string param; int index; double q, sig, eps; };
    void readForce(const NonbondedForce& force) {
        const int n = force.getNumParticles();
        baseQ.resize(n); baseSig.resize(n); baseEps.resize(n);
        for (int i = 0; i < n; i++) force.getParticleParameters(i, baseQ[i], baseSig[i], baseEps[i]);
        const int ne = force.getNumExceptions();
        ei.resize(ne); ej.resize(ne); baseEqq.resize(ne); baseEsig.resize(ne); baseEeps.resize(ne);
        for (int e = 0; e < ne; e++) force.getExceptionParameters(e, ei[e], ej[e], baseEqq[e], baseEsig[e], baseEeps[e]);
        particleOffsets.clear(); exceptionOffsets.clear(); paramNames.clear();
        for (int i = 0; i < force.getNumParticleParameterOffsets(); i++) {
            Offset o; force.getParticleParameterOffset(i, o.param, o.index, o.q, o.sig, o.eps);
            particleOffsets.push_back(o); paramNames[o.param] = 0.0;
        }
        for (int i = 0; i < force.getNumExceptionParameterOffsets(); i++) {
            Offset o; force.getExceptionParameterOffset(i, o.param, o.index, o.q, o.sig, o.eps);
            exceptionOffsets.push_back(o); paramNames[o.param] = 0.0;
        }
    }
    // computeParameters of the reference (ReferenceKernels.cpp:1077-1121): parameter = base + sum(scale * global value)
    void effective(const map<string, double>& value, vector<double>& q, vector<double>& sig, vector<double>& eps,
                   vector<double>& eqq, vector<double>& esig, vector<double>& eeps) const {
        q = baseQ; sig = baseSig; eps = baseEps; eqq = baseEqq; esig = baseEsig; eeps = baseEeps;
        for (const Offset& o : particleOffsets) { const double v = value.at(o.param); q[o.index] += v*o.q; sig[o.index] += v*o.sig; eps[o.index] += v*o.eps; }
        for (const Offset& o : exceptionOffsets) { const double v = value.at(o.param); eqq[o.index] += v*o.q; esig[o.index] += v*o.sig; eeps[o.index] += v*o.eps; }
    }
    void initialize(const System& system, const NonbondedForce& force) {
        PlatformData& d = getData(context);
        if (d.finalized) throw OpenMMException("B200 platform: NonbondedForce initialised after the Context was finalised");
        b200md_nonbonded_desc nd;
        nd.method = (int) force.getNonbondedMethod();
        if (nd.method == B200MD_NB_EWALD || nd.method == B200MD_NB_LJPME)
            throw OpenMMException("B200 platform: only NoCutoff, CutoffNonPeriodic, CutoffPeriodic and PME are supported");
        nd.cutoff = force.getCutoffDistance();
        nd.use_switch = force.getUseSwitchingFunction() ? 1 : 0;
        nd.switch_distance = force.getSwitchingDistance();
        nd.rf_dielectric = force.getReactionFieldDielectric();
        nd.ewald_alpha = 0; nd.grid[0] = nd.grid[1] = nd.grid[2] = 0;
        if (nd.method == B200MD_NB_PME) {
            NonbondedForceImpl::calcPMEParameters(system, force, alpha, grid[0], grid[1], grid[2], false);
            for (int k = 0; k < 3; k++) grid[k] = fftFriendly(grid[k]);
            nd.ewald_alpha = alpha;
            for (int k = 0; k < 3; k++) nd.grid[k] = grid[k];
        }
        // platform-independent static helper of the reference: call it, don't rewrite it (SURVEY.md a16)
        nd.dispersion_coefficient = force.getUseDispersionCorrection() ? NonbondedForceImpl::calcDispersionCorrection(system, force) : 0.0;
        nd.exceptions_periodic = force.getExceptionsUsePeriodicBoundaryConditions() ? 1 : 0;
        readForce(force);
        // the Context's parameter map does not exist yet (ContextImpl.cpp:120-131 fills it after the kernels are
        // initialised): start from the defaults, execute() re-uploads whenever a value differs
        for (int i = 0; i < force.getNumGlobalParameters(); i++)
            if (paramNames.count(force.getGlobalParameterName(i))) paramNames[force.getGlobalParameterName(i)] = force.getGlobalParameterDefaultValue(i);
        vector<double> q, sig, eps, eqq, esig, eeps;
        effective(paramNames, q, sig, eps, eqq, esig, eeps);
        d.check(b200md_set_nonbonded(d.ctx, &nd, q.data(), sig.data(), eps.data()));
        if (!ei.empty()) d.check(b200md_set_exceptions(d.ctx, (int) ei.size(), ei.data(), ej.data(), eqq.data(), esig.data(), eeps.data()));
        dispersion = nd.dispersion_coefficient;
        d.systemTerms |= B200MD_TERM_NB_DIRECT | B200MD_TERM_NB_RECIP;
    }
    void upload(PlatformData& d) {
        vector<double> q, sig, eps, eqq, esig, eeps;
        effective(paramNames, q, sig, eps, eqq, esig, eeps);
        d.check(b200md_update_nonbonded_params(d.ctx, q.data(), sig.data(), eps.data(), (int) ei.size(), eqq.data(), esig.data(), eeps.data(), dispersion));
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy, bool includeDirect, bool includeReciprocal) {
        PlatformData& d = getData(context);
        if (!paramNames.empty()) {
            bool changed = false;
            for (auto& pv : paramNames) {
                const double v = context.getParameter(pv.first);
                if (v != pv.second) { pv.second = v; changed = true; }
            }
            if (changed) upload(d);
        }
        if (includeDirect) d.pendingTerms |= B200MD_TERM_NB_DIRECT;
        if (includeReciprocal) d.pendingTerms |= B200MD_TERM_NB_RECIP;
        return 0.0;     // the energy comes back through finishComputation
    }
    void copyParametersToContext(ContextImpl& context, const NonbondedForce& force) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        if (force.getNumParticles() != (int) baseQ.size()) throw OpenMMException("updateParametersInContext: The number of particles has changed");
        if (force.getNumExceptions() != (int) ei.size()) throw OpenMMException("updateParametersInContext: The number of exceptions has changed");
        const vector<int> oi = ei, oj = ej;
        const map<string, double> old = paramNames;
        readForce(force);
        for (size_t e = 0; e < ei.size(); e++)
            if (ei[e] != oi[e] || ej[e] != oj[e]) throw OpenMMException("updateParametersInContext: The set of particles in an exception has changed");
        for (auto& pv : paramNames) pv.second = context.getParameter(pv.first);
        dispersion = force.getUseDispersionCorrection() ? NonbondedForceImpl::calcDispersionCorrection(context.getSystem(), force) : 0.0;
        upload(d);
    }
    void getPMEParameters(double& a, int& nx, int& ny, int& nz) const { a = alpha; nx = grid[0]; ny = grid[1]; nz = grid[2]; }
    void getLJPMEParameters(double& a, int& nx, int& ny, int& nz) const { throw OpenMMException("B200 platform: LJPME is not supported"); }
private:
    ContextImpl& context;
    double alpha, dispersion = 0;
    int grid[3];
    vector<double> baseQ, baseSig, baseEps, baseEqq, baseEsig, baseEeps;
    vector<int> ei, ej;
    vector<Offset> particleOffsets, exceptionOffsets;
    map<string, double> paramNames;      // global parameters used by offsets -> value the device parameters were computed with
};

// Bonded forces: any number of Force objects per class.  Every object appends its terms (tagged with its force group) to
// its class's TermRecord; the engine evaluates a term iff its class was executed in this evaluation AND its group is in
// the `groups` mask of finishComputation (ForceImpl::calcForcesAndEnergy only calls execute for objects whose group is in it).
// ObjectTerms is what every bonded kernel shares: this object's terms are [first, first+count) of the record.  read(i, r)
// appends term i of the object to r; the same reader fills the record at initialize and re-reads the object on update.
class ObjectTerms {
protected:
    int first = 0, count = 0;
    template<class Read> void add(PlatformData& d, TermRecord& r, const Force& force, int numTerms, int bit, const char* name, Read read) {
        if (d.finalized) throw OpenMMException(string("B200 platform: ") + name + " initialised after the Context was finalised");
        first = r.size(); count = numTerms;
        for (int i = 0; i < count; i++) read(i, r);
        r.group.resize(first + count, force.getForceGroup() | (force.usesPeriodicBoundaryConditions() ? 0x80 : 0));
        d.systemTerms |= bit; d.bondedGroupsUsed |= 1u << force.getForceGroup();
    }
    // copyParametersToContext: the object read again, refused if the number of its terms or the atoms of one changed
    template<class Read> TermRecord reread(PlatformData& d, const TermRecord& r, int numTerms, const char* terms, const char* aTerm, Read read) const {
        d.ensureFinalized();
        d.dropForces();
        if (numTerms != count) throw OpenMMException(string("updateParametersInContext: The number of ") + terms + " has changed");
        TermRecord fresh(r.kind, r.atoms.size(), r.ints.size(), r.params.size());
        for (int i = 0; i < count; i++) read(i, fresh);
        for (size_t c = 0; c < r.atoms.size(); c++)
            if (!equal(fresh.atoms[c].begin(), fresh.atoms[c].end(), start(r.atoms[c], r)))
                throw OpenMMException(string("updateParametersInContext: The set of particles in ") + aTerm + " has changed");
        return fresh;
    }
    // the parameters of `fresh` (reread) into [first, first+count)
    void store(TermRecord& r, const TermRecord& fresh) const {
        for (size_t c = 0; c < r.ints.size(); c++) copy(fresh.ints[c].begin(), fresh.ints[c].end(), start(r.ints[c], r));
        for (size_t c = 0; c < r.params.size(); c++) copy(fresh.params[c].begin(), fresh.params[c].end(), start(r.params[c], r));
    }
private:
    // where this object's terms start in a column of r
    template<class V> auto start(V& column, const TermRecord& r) const -> decltype(column.begin()) {
        return column.begin() + (count ? column.size()/r.size()*first : 0);
    }
};

// HarmonicBondForce, HarmonicAngleForce, PeriodicTorsionForce and RBTorsionForce (T: Bonds, Angles, Torsions, RBTorsions)
template<class T, TermRecord PlatformData::* record>
class B200CalcBondedForceKernel : public T::Kernel, ObjectTerms {
public:
    B200CalcBondedForceKernel(string name, const Platform& platform, ContextImpl& context) : T::Kernel(name, platform), context(context) {}
    void initialize(const System& system, const typename T::Force& force) {
        PlatformData& d = getData(context);
        add(d, d.*record, force, T::count(force), T::bit, T::name, [&](int i, TermRecord& r) { T::read(force, i, r); });
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) { getData(context).pendingTerms |= T::bit; return 0.0; }
    void copyParametersToContext(ContextImpl& context, const typename T::Force& force) {
        PlatformData& d = getData(context);
        TermRecord& r = d.*record;
        store(r, reread(d, r, T::count(force), T::terms, T::aTerm, [&](int i, TermRecord& f) { T::read(force, i, f); }));
        d.check(T::update(d.ctx, r));
    }
private:
    ContextImpl& context;
};

// The library takes spline coefficients: the reference's own platform-independent fitter makes them (call, don't rewrite).
class B200CalcCMAPTorsionForceKernel : public CalcCMAPTorsionForceKernel, ObjectTerms {
public:
    B200CalcCMAPTorsionForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcCMAPTorsionForceKernel(name, platform), context(context) {}
    // the coefficients of the maps of `force`, appended to coeff; their sizes appended to size
    static void readMaps(const CMAPTorsionForce& force, vector<int>& size, vector<double>& coeff) {
        vector<double> energy;
        vector<vector<double> > c;
        for (int m = 0; m < force.getNumMaps(); m++) {
            int n;
            force.getMapParameters(m, n, energy);
            CMAPTorsionForceImpl::calcMapDerivatives(n, energy, c);
            size.push_back(n);
            for (const vector<double>& patch : c) coeff.insert(coeff.end(), patch.begin(), patch.end());
        }
    }
    void read(const CMAPTorsionForce& force, int i, TermRecord& r) const {
        int m, a[8];
        force.getTorsionParameters(i, m, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);
        r.add(vector<int>(a, a + 8), {firstMap + m}, {});
    }
    void initialize(const System& system, const CMAPTorsionForce& force) {
        PlatformData& d = getData(context);
        firstMap = (int) d.cmapSize.size(); numMaps = force.getNumMaps();
        firstCoeff = d.cmapCoeff.size();
        add(d, d.cmap, force, force.getNumTorsions(), B200MD_TERM_CMAP, "CMAPTorsionForce", [&](int i, TermRecord& r) { read(force, i, r); });
        readMaps(force, d.cmapSize, d.cmapCoeff);
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) { getData(context).pendingTerms |= B200MD_TERM_CMAP; return 0.0; }
    void copyParametersToContext(ContextImpl& context, const CMAPTorsionForce& force) {
        PlatformData& d = getData(context);
        if (force.getNumMaps() != numMaps) throw OpenMMException("updateParametersInContext: The number of maps has changed");
        const TermRecord fresh = reread(d, d.cmap, force.getNumTorsions(), "CMAP torsions", "a CMAP torsion", [&](int i, TermRecord& r) { read(force, i, r); });
        vector<int> size;
        vector<double> coeff;
        readMaps(force, size, coeff);
        for (int m = 0; m < numMaps; m++)
            if (size[m] != d.cmapSize[firstMap+m]) throw OpenMMException("updateParametersInContext: The size of a map has changed");
        for (int m : fresh.ints[0])
            if (m < firstMap || m >= firstMap + numMaps) throw OpenMMException("updateParametersInContext: CMAP torsion map index out of range");
        store(d.cmap, fresh);
        copy(coeff.begin(), coeff.end(), d.cmapCoeff.begin() + firstCoeff);
        d.check(b200md_update_cmap_params(d.ctx, (int) d.cmapSize.size(), d.cmapSize.data(), d.cmapCoeff.data(), d.cmap.size(), d.cmap.ints[0].data()));
    }
private:
    ContextImpl& context;
    int firstMap = 0, numMaps = 0;
    size_t firstCoeff = 0;
};

// CustomTorsionForce: the expression becomes two instruction programs (custom_translate.h), which k_custom_torsion interprets.
vector<string> perTorsionParameterNames(const CustomTorsionForce& force) {
    vector<string> names;
    for (int i = 0; i < force.getNumPerTorsionParameters(); i++) names.push_back(force.getPerTorsionParameterName(i));
    return names;
}
vector<string> globalParameterNames(const CustomTorsionForce& force) {
    vector<string> names;
    for (int i = 0; i < force.getNumGlobalParameters(); i++) names.push_back(force.getGlobalParameterName(i));
    return names;
}

class B200CalcCustomTorsionForceKernel : public CalcCustomTorsionForceKernel, ObjectTerms {
public:
    B200CalcCustomTorsionForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcCustomTorsionForceKernel(name, platform), context(context) {}
    // the term's parameters: as many as the force declares (the Reference platform reads as many), padded with zeros
    void read(const CustomTorsionForce& force, int i, TermRecord& r) const {
        int a, b, c, e;
        vector<double> par;
        force.getTorsionParameters(i, a, b, c, e, par);
        par.resize(numParams);
        par.resize(B200MD_CUSTOM_MAX_PARAMS, 0.0);
        r.add({a, b, c, e}, {prog}, par);
    }
    void initialize(const System& system, const CustomTorsionForce& force) {
        PlatformData& d = getData(context);
        prog = (int) d.customProgStart.size()/2;
        numParams = force.getNumPerTorsionParameters();
        add(d, d.custom, force, force.getNumTorsions(), B200MD_TERM_CUSTOM_TORSIONS, "CustomTorsionForce", [&](int i, TermRecord& r) { read(force, i, r); });
        b200md_custom::Program energy, deriv;
        const vector<string> globals = globalParameterNames(force);
        b200md_custom::translateExpression(force.getEnergyFunction(), perTorsionParameterNames(force), globals, d.customGlobalSlot, energy, deriv);
        for (const b200md_custom::Program* p : {&energy, &deriv}) {
            d.customOp.insert(d.customOp.end(), p->op.begin(), p->op.end());
            d.customArg.insert(d.customArg.end(), p->arg.begin(), p->arg.end());
            d.customImm.insert(d.customImm.end(), p->imm.begin(), p->imm.end());
            d.customProgStart.push_back((int) d.customOp.size());
        }
        // the Context's parameter map does not exist yet (ContextImpl.cpp:120-131 fills it after the kernels are initialised):
        // start from the defaults, execute() sends whatever differs
        d.customGlobals.resize(d.customGlobalSlot.size(), 0.0);
        for (int i = 0; i < force.getNumGlobalParameters(); i++) {
            const map<string, int>::const_iterator it = d.customGlobalSlot.find(force.getGlobalParameterName(i));
            if (it == d.customGlobalSlot.end()) continue;         // declared, but the expression does not read it
            slots.push_back(make_pair(it->first, it->second));
            d.customGlobals[it->second] = force.getGlobalParameterDefaultValue(i);
        }
        d.customStride = max(d.customStride, numParams);
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) {
        PlatformData& d = getData(context);
        // a changed global value is a stream-ordered copy into the buffer the step graph reads (NonbondedForce offsets alike)
        bool changed = false;
        for (const pair<string, int>& s : slots) {
            const double v = context.getParameter(s.first);
            if (v != d.customGlobals[s.second]) { d.customGlobals[s.second] = v; changed = true; }
        }
        if (changed) d.check(b200md_set_custom_globals(d.ctx, (int) d.customGlobals.size(), d.customGlobals.data()));
        d.pendingTerms |= B200MD_TERM_CUSTOM_TORSIONS;
        return 0.0;
    }
    void copyParametersToContext(ContextImpl& context, const CustomTorsionForce& force) {
        PlatformData& d = getData(context);
        store(d.custom, reread(d, d.custom, force.getNumTorsions(), "torsions", "a torsion", [&](int i, TermRecord& r) { read(force, i, r); }));
        const vector<double> packed = d.packedCustomParams();
        d.check(b200md_update_custom_torsion_params(d.ctx, d.custom.size(), packed.data()));
    }
private:
    ContextImpl& context;
    int prog = 0, numParams = 0;          // this object's program pair; its number of per-torsion parameters
    vector<pair<string, int> > slots;     // the global parameters this object's expression reads, and their slots
};

// RemoveCMMotionKernel::execute is called by CMMotionRemoverImpl::updateContextState in EVERY step; the frequency test is
// the kernel's (ReferenceKernels.cpp:2712-2714).  The removal itself is deferred to the integrator step that follows (the
// fused step graph removes the centre-of-mass motion itself) or to the next read of the velocities (PlatformData::flushCm).
class B200RemoveCMMotionKernel : public RemoveCMMotionKernel {
public:
    B200RemoveCMMotionKernel(string name, const Platform& platform, ContextImpl& context) : RemoveCMMotionKernel(name, platform), context(context) {}
    void initialize(const System& system, const CMMotionRemover& force) {
        PlatformData& d = getData(context);
        d.cmFrequency = force.getFrequency();
        d.check(b200md_set_cm_remover(d.ctx, d.cmFrequency));
    }
    void execute(ContextImpl& context) { PlatformData& d = getData(context); d.ensureFinalized(); d.cmRequested = true; }
private:
    ContextImpl& context;
};

// ------------------------------------------------------------------------------------------------ integrators
// The reference's Integrator::step drives updateContextState -> calcForcesAndEnergy -> kernel.execute per step
// (LangevinIntegrator.cpp:74-82); execute() is the integrate+constrain half, enqueued with no host sync.
void configureIntegrator(ContextImpl& context, int kind, double dt, double temperature, double friction, int seed, double tol) {
    PlatformData& d = getData(context);
    if (d.integratorKind == kind && d.dt == dt && d.temperature == temperature && d.friction == friction && d.tol == tol && d.seed == seed) return;
    d.check(b200md_set_integrator(d.ctx, kind, dt, temperature, friction, seed, tol));
    d.integratorKind = kind; d.dt = dt; d.temperature = temperature; d.friction = friction; d.tol = tol; d.seed = seed;
}

// The integrate + constrain half of a step.  When the forces-only evaluation that precedes it in Integrator::step is still
// pending and covered the whole force field, forces + integration run as ONE replay of the captured step graph.
void integrateStep(ContextImpl& context) {
    PlatformData& d = getData(context);
    d.checkBox();
    d.ensureFinalized();
    const bool whole = d.lazyForces && d.lazyTerms == d.systemTerms && (d.bondedGroupsUsed & ~d.lazyGroups) == 0;
    if (whole && d.useFusedStep) {
        d.lazyForces = false; d.cmRequested = false;         // b200md_step removes the centre-of-mass motion at its own frequency
        d.check(b200md_step(d.ctx, 1));
        return;
    }
    d.flushCm();
    d.flushForces();
    d.check(b200md_integrate_only(d.ctx));
}
double kineticEnergy(ContextImpl& context) {
    PlatformData& d = getData(context);
    d.ensureFinalized();
    d.flushCm();
    d.flushForces();         // the leapfrog integrators report the kinetic energy at a half-step-shifted velocity (ReferenceKernels.cpp:146-176)
    double ke = 0; d.check(b200md_kinetic_energy(d.ctx, &ke)); return ke;
}

class B200IntegrateVerletStepKernel : public IntegrateVerletStepKernel {
public:
    B200IntegrateVerletStepKernel(string name, const Platform& platform) : IntegrateVerletStepKernel(name, platform) {}
    void initialize(const System& system, const VerletIntegrator& integrator) {}
    void configure(ContextImpl& context, const VerletIntegrator& in) { configureIntegrator(context, B200MD_INT_VERLET, in.getStepSize(), 0.0, 0.0, 0, in.getConstraintTolerance()); }
    void execute(ContextImpl& context, const VerletIntegrator& integrator) { configure(context, integrator); integrateStep(context); }
    double computeKineticEnergy(ContextImpl& context, const VerletIntegrator& integrator) { configure(context, integrator); return kineticEnergy(context); }
};

class B200IntegrateLangevinStepKernel : public IntegrateLangevinStepKernel {
public:
    B200IntegrateLangevinStepKernel(string name, const Platform& platform) : IntegrateLangevinStepKernel(name, platform) {}
    void initialize(const System& system, const LangevinIntegrator& integrator) {}
    void configure(ContextImpl& context, const LangevinIntegrator& in) {
        configureIntegrator(context, B200MD_INT_LANGEVIN, in.getStepSize(), in.getTemperature(), in.getFriction(), in.getRandomNumberSeed(), in.getConstraintTolerance());
    }
    void execute(ContextImpl& context, const LangevinIntegrator& integrator) { configure(context, integrator); integrateStep(context); }
    double computeKineticEnergy(ContextImpl& context, const LangevinIntegrator& integrator) { configure(context, integrator); return kineticEnergy(context); }
};

class B200IntegrateLangevinMiddleStepKernel : public IntegrateLangevinMiddleStepKernel {
public:
    B200IntegrateLangevinMiddleStepKernel(string name, const Platform& platform) : IntegrateLangevinMiddleStepKernel(name, platform) {}
    void initialize(const System& system, const LangevinMiddleIntegrator& integrator) {}
    void configure(ContextImpl& context, const LangevinMiddleIntegrator& in) {
        configureIntegrator(context, B200MD_INT_LANGEVIN_MIDDLE, in.getStepSize(), in.getTemperature(), in.getFriction(), in.getRandomNumberSeed(), in.getConstraintTolerance());
    }
    void execute(ContextImpl& context, const LangevinMiddleIntegrator& integrator) { configure(context, integrator); integrateStep(context); }
    double computeKineticEnergy(ContextImpl& context, const LangevinMiddleIntegrator& integrator) { configure(context, integrator); return kineticEnergy(context); }
};

// ------------------------------------------------------------------------------------------------ barostat
// MonteCarloBarostat / MonteCarloAnisotropicBarostat: MonteCarloBarostatImpl (the reference's, untouched) draws the move, evaluates
// the energy before and after, and accepts or rejects; the platform scales the molecules and restores them on rejection.
class B200ApplyMonteCarloBarostatKernel : public ApplyMonteCarloBarostatKernel {
public:
    B200ApplyMonteCarloBarostatKernel(string name, const Platform& platform) : ApplyMonteCarloBarostatKernel(name, platform) {}
    void initialize(const System& system, const Force& barostat) {}
    void scaleCoordinates(ContextImpl& context, double scaleX, double scaleY, double scaleZ) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        if (!haveMolecules) {
            // ContextImpl::getMolecules() exists only once every ForceImpl is initialised: upload it at the first move, as
            // CommonApplyMonteCarloBarostatKernel::scaleCoordinates does
            const vector<vector<int> >& mols = context.getMolecules();
            vector<int> start(1, 0), atoms;
            for (const vector<int>& m : mols) { atoms.insert(atoms.end(), m.begin(), m.end()); start.push_back((int) atoms.size()); }
            d.check(b200md_set_barostat_molecules(d.ctx, (int) mols.size(), start.data(), atoms.data()));
            haveMolecules = true;
        }
        d.check(b200md_scale_coordinates(d.ctx, scaleX, scaleY, scaleZ));
    }
    void restoreCoordinates(ContextImpl& context) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        d.check(b200md_restore_coordinates(d.ctx));
    }
private:
    bool haveMolecules = false;
};

// ------------------------------------------------------------------------------------------------ factory + platform
class B200KernelFactory : public KernelFactory {
public:
    KernelImpl* createKernelImpl(string name, const Platform& platform, ContextImpl& context) const {
        if (name == CalcForcesAndEnergyKernel::Name()) return new B200CalcForcesAndEnergyKernel(name, platform);
        if (name == UpdateStateDataKernel::Name()) return new B200UpdateStateDataKernel(name, platform);
        if (name == ApplyConstraintsKernel::Name()) return new B200ApplyConstraintsKernel(name, platform);
        if (name == VirtualSitesKernel::Name()) return new B200VirtualSitesKernel(name, platform);
        if (name == CalcNonbondedForceKernel::Name()) return new B200CalcNonbondedForceKernel(name, platform, context);
        if (name == CalcHarmonicBondForceKernel::Name()) return new B200CalcBondedForceKernel<Bonds, &PlatformData::bonds>(name, platform, context);
        if (name == CalcHarmonicAngleForceKernel::Name()) return new B200CalcBondedForceKernel<Angles, &PlatformData::angles>(name, platform, context);
        if (name == CalcPeriodicTorsionForceKernel::Name()) return new B200CalcBondedForceKernel<Torsions, &PlatformData::torsions>(name, platform, context);
        if (name == CalcRBTorsionForceKernel::Name()) return new B200CalcBondedForceKernel<RBTorsions, &PlatformData::rb>(name, platform, context);
        if (name == CalcCMAPTorsionForceKernel::Name()) return new B200CalcCMAPTorsionForceKernel(name, platform, context);
        if (name == CalcCustomTorsionForceKernel::Name()) return new B200CalcCustomTorsionForceKernel(name, platform, context);
        if (name == RemoveCMMotionKernel::Name()) return new B200RemoveCMMotionKernel(name, platform, context);
        if (name == IntegrateVerletStepKernel::Name()) return new B200IntegrateVerletStepKernel(name, platform);
        if (name == IntegrateLangevinStepKernel::Name()) return new B200IntegrateLangevinStepKernel(name, platform);
        if (name == IntegrateLangevinMiddleStepKernel::Name()) return new B200IntegrateLangevinMiddleStepKernel(name, platform);
        if (name == ApplyMonteCarloBarostatKernel::Name()) return new B200ApplyMonteCarloBarostatKernel(name, platform);
        throw OpenMMException((string("Tried to create kernel with illegal kernel name '") + name + "'").c_str());
    }
};

class B200Platform : public Platform {
public:
    B200Platform() {
        B200KernelFactory* factory = new B200KernelFactory();
        for (const string& n : {CalcForcesAndEnergyKernel::Name(), UpdateStateDataKernel::Name(), ApplyConstraintsKernel::Name(), VirtualSitesKernel::Name(),
                                CalcNonbondedForceKernel::Name(), CalcHarmonicBondForceKernel::Name(), CalcHarmonicAngleForceKernel::Name(),
                                CalcPeriodicTorsionForceKernel::Name(), CalcRBTorsionForceKernel::Name(), CalcCMAPTorsionForceKernel::Name(),
                                CalcCustomTorsionForceKernel::Name(), RemoveCMMotionKernel::Name(), IntegrateVerletStepKernel::Name(),
                                IntegrateLangevinStepKernel::Name(), IntegrateLangevinMiddleStepKernel::Name(), ApplyMonteCarloBarostatKernel::Name()})
            registerKernelFactory(n, factory);
        platformProperties.push_back(DeviceIndex());
        platformProperties.push_back(Precision());
        setPropertyDefaultValue(DeviceIndex(), "0");
        setPropertyDefaultValue(Precision(), "single");
    }
    static const string& DeviceIndex() { static const string key = "DeviceIndex"; return key; }
    static const string& Precision() { static const string key = "Precision"; return key; }
    const string& getName() const { static const string name = "B200"; return name; }
    double getSpeed() const { return 200; }        // CUDA = 100 (CudaPlatform.cpp:149-151): win auto-selection; what this platform cannot run is refused in contextCreated
    bool supportsDoublePrecision() const { return false; }
    const string& getPropertyValue(const Context& context, const string& property) const {
        const ContextImpl& impl = getContextImpl(context);
        const PlatformData& d = getData(impl);
        map<string, string>::const_iterator it = d.props.find(property);
        if (it != d.props.end()) return it->second;
        return Platform::getPropertyValue(context, property);
    }
    void setPropertyValue(Context& context, const string& property, const string& value) const {
        // no property of this platform can change once the Context exists (DeviceIndex and Precision are fixed at creation)
        throw OpenMMException("B200 platform: property '" + property + "' cannot be changed after the Context was created");
    }
    // Everything the kernels would refuse LATER must be refused HERE: ContextImpl only falls back to the next platform
    // when contextCreated() throws (ContextImpl.cpp:152-166); a throw from Kernel::initialize or from the first
    // setPositions would instead make Context creation fail for a System that CUDA / CPU can run.
    static void validateSystem(const System& system) {
        for (int i = 0; i < system.getNumParticles(); i++)
            if (system.isVirtualSite(i)) throw OpenMMException("B200 platform: virtual sites are not supported");
        int numNonbonded = 0;
        for (int f = 0; f < system.getNumForces(); f++) {
            const Force& force = system.getForce(f);
            if (const NonbondedForce* nb = dynamic_cast<const NonbondedForce*>(&force)) {
                if (++numNonbonded > 1) throw OpenMMException("B200 platform: only one NonbondedForce per System is supported");
                const NonbondedForce::NonbondedMethod m = nb->getNonbondedMethod();
                if (m == NonbondedForce::Ewald || m == NonbondedForce::LJPME)
                    throw OpenMMException("B200 platform: only NoCutoff, CutoffNonPeriodic, CutoffPeriodic and PME are supported");
                if (nb->getNumParticles() != system.getNumParticles()) throw OpenMMException("NonbondedForce must have exactly as many particles as the System it belongs to.");
            }
            if (force.getForceGroup() < 0 || force.getForceGroup() > 31) throw OpenMMException("B200 platform: force group out of range");
            if (dynamic_cast<const MonteCarloMembraneBarostat*>(&force)) throw OpenMMException("B200 platform: MonteCarloMembraneBarostat is not supported");
            if (const CustomTorsionForce* ct = dynamic_cast<const CustomTorsionForce*>(&force)) {
                // getEnergyParameterDerivatives returns nothing here
                if (ct->getNumEnergyParameterDerivatives() > 0) throw OpenMMException("B200 platform: energy parameter derivatives of a CustomTorsionForce are not supported");
                // beyond the interpreter's limits: refused here; an unknown variable is an error on every platform and is
                // raised by the kernel's initialize, as the Reference platform does
                map<string, int> slots;
                b200md_custom::Program e, de;
                try { b200md_custom::translateExpression(ct->getEnergyFunction(), perTorsionParameterNames(*ct), globalParameterNames(*ct), slots, e, de); }
                catch (const b200md_custom::Unsupported&) { throw; }
                catch (const OpenMMException&) {}
            }
        }
        const int nc = system.getNumConstraints();
        if (nc > 0) {
            vector<int> ci(nc), cj(nc); vector<double> cd(nc), mass(system.getNumParticles());
            for (int k = 0; k < nc; k++) system.getConstraintParameters(k, ci[k], cj[k], cd[k]);
            for (int i = 0; i < system.getNumParticles(); i++) mass[i] = system.getParticleMass(i);
            char msg[256];
            if (b200md_check_constraints(system.getNumParticles(), mass.data(), nc, ci.data(), cj.data(), cd.data(), msg, sizeof(msg)) != 0)
                throw OpenMMException(string("B200 platform: ") + msg);
        }
    }
    void contextCreated(ContextImpl& context, const map<string, string>& properties) const {
        validateSystem(context.getSystem());
        PlatformData* d = new PlatformData();
        if (getenv("B200MD_PLUGIN_FUSED")) d->useFusedStep = atoi(getenv("B200MD_PLUGIN_FUSED")) != 0;
        try {
            string dev = properties.count(DeviceIndex()) ? properties.at(DeviceIndex()) : getPropertyDefaultValue(DeviceIndex());
            string prec = properties.count(Precision()) ? properties.at(Precision()) : getPropertyDefaultValue(Precision());
            // mixed: positions hi + lo, velocities, integration and constraints in double, forces in single precision (the
            // reference GPU platforms' definition).  double is refused here, so OpenMM moves such a Context to another platform.
            if (prec != "single" && prec != "mixed") throw OpenMMException("B200 platform: Precision=" + prec + " is not supported (single or mixed)");
            const System& system = context.getSystem();
            d->numParticles = system.getNumParticles();
            if (b200md_create(&d->ctx, atoi(dev.c_str()), d->numParticles) != 0)
                throw OpenMMException(string("B200 platform: ") + b200md_last_error(nullptr));
            d->props[DeviceIndex()] = dev;
            d->props[Precision()] = prec;
            d->check(b200md_set_precision(d->ctx, prec == "mixed" ? B200MD_PRECISION_MIXED : B200MD_PRECISION_SINGLE));
            vector<double> mass(d->numParticles);
            for (int i = 0; i < d->numParticles; i++) mass[i] = system.getParticleMass(i);
            d->check(b200md_set_masses(d->ctx, mass.data()));
            const int nc = system.getNumConstraints();
            if (nc > 0) {
                vector<int> ci(nc), cj(nc); vector<double> cd(nc);
                for (int k = 0; k < nc; k++) system.getConstraintParameters(k, ci[k], cj[k], cd[k]);
                d->check(b200md_set_constraints(d->ctx, nc, ci.data(), cj.data(), cd.data()));
            }
        } catch (...) {
            if (d->ctx) b200md_destroy(d->ctx);
            delete d;
            throw;
        }
        context.setPlatformData(d);
    }
    void contextDestroyed(ContextImpl& context) const {
        PlatformData* d = reinterpret_cast<PlatformData*>(context.getPlatformData());
        if (d) { if (d->ctx) b200md_destroy(d->ctx); delete d; }
    }
};

} // namespace

extern "C" __attribute__((visibility("default"))) void registerPlatforms() {
    Platform::registerPlatform(new B200Platform());
}

extern "C" __attribute__((visibility("default"))) void registerKernelFactories() {
}
