// B200Platform.cpp -- libOpenMMB200.so: the OpenMM Platform plugin for the CUDA-native (sm_90a) hot path.
//
// A thin C++ adapter: every KernelImpl below forwards one abstract kernel interface of the reference
// (olla/include/openmm/kernels.h) to the C-ABI of libb200md.so (include/b200md.h), where all the CUDA lives.
// Loaded by Platform::loadPluginLibrary / loadPluginsFromDirectory (olla/src/Platform.cpp:221-320) through the
// extern "C" registerPlatforms() entry point (PluginInitializer.h:47), exactly like platforms/cuda
// (CudaPlatform.cpp:59-61).  Compiled against the reference's headers where they lie; no reference source is copied.
//
// Supported: NonbondedForce (NoCutoff, CutoffNonPeriodic, CutoffPeriodic, PME; parameter offsets), HarmonicBondForce,
// HarmonicAngleForce, PeriodicTorsionForce, RBTorsionForce, CMAPTorsionForce, CustomTorsionForce, CustomBondForce,
// CustomExternalForce, CustomAngleForce, CustomCompoundBondForce, CustomCentroidBondForce (any number of objects, each in its own force group; custom forces without energy parameter
// derivatives, expressions within the limits of custom_translate.h), GBSAOBCForce (one per System, its method and cutoff
// matching the NonbondedForce's; NoCutoff also without one), RMSDForce (any number of objects), CustomNonbondedForce (any
// number of objects sharing one method, cutoff and exclusion set, which are the NonbondedForce's when there is one; discrete
// tables, switching function, long-range correction; no interaction groups), CMMotionRemover;
// Verlet / Langevin / LangevinMiddle integrators; SETTLE + X-H_n SHAKE constraints; MonteCarloBarostat and
// MonteCarloAnisotropicBarostat (ApplyMonteCarloBarostatKernel; MonteCarloMembraneBarostat is refused).  A Force class without a kernel here
// makes Platform::supportsKernels() false; an unsupported OPTION of a supported class is rejected in contextCreated()
// (validateSystem), which is the only place from which ContextImpl falls back to the next platform (ContextImpl.cpp:152-166).
//
// Bonded classes.  Each keeps the terms of all its Force objects in one TermRecord of PlatformData, sent at finalize; what
// their kernels share (ObjectTerms: the object's range of the record, group tags, updates) exists once.  Bond, angle,
// periodic-torsion and RB-torsion kernels are one template, B200CalcBondedForceKernel; the custom torsion, bond, external,
// angle, compound-bond and centroid-bond kernels another, B200CalcCustomForceKernel, for their expression programs; CMAP keeps its own for
// its maps.
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
#include "openmm/CustomBondForce.h"
#include "openmm/CustomExternalForce.h"
#include "openmm/CustomAngleForce.h"
#include "openmm/CustomCompoundBondForce.h"
#include "openmm/CustomCentroidBondForce.h"
#include "openmm/GBSAOBCForce.h"
#include "openmm/RMSDForce.h"
#include "openmm/CustomCVForce.h"
#include "openmm/CustomNonbondedForce.h"
#include "openmm/internal/CustomNonbondedForceImpl.h"
#include "openmm/TabulatedFunction.h"
#include "lepton/CustomFunction.h"
#include "lepton/ExpressionProgram.h"
#include "lepton/ParsedExpression.h"
#include "lepton/Parser.h"
#include "openmm/CMMotionRemover.h"
#include "openmm/VerletIntegrator.h"
#include "openmm/LangevinIntegrator.h"
#include "openmm/LangevinMiddleIntegrator.h"
#include "openmm/MonteCarloMembraneBarostat.h"
#include "openmm/internal/ContextImpl.h"
#include "openmm/internal/NonbondedForceImpl.h"
#include "openmm/internal/CMAPTorsionForceImpl.h"
#include "openmm/internal/CustomCentroidBondForceImpl.h"
#include "../include/b200md.h"
#include "custom_translate.h"
#include <algorithm>
#include <map>
#include <set>
#include <string>
#include <vector>
#include <sstream>
#include <cstdlib>

using namespace OpenMM;
using namespace std;

// the Reference platform's spline of a TabulatedFunction as a Lepton function, exported by libOpenMM.so
// (platforms/reference/include/ReferenceTabulatedFunction.h)
extern "C" Lepton::CustomFunction* createReferenceTabulatedFunction(const TabulatedFunction& function);

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

// The expression programs of one custom class over all its Force objects, one after the other (object f's expression is
// expression f); per expression its first program, its particles per term and whether its point functions take the minimum
// image (both 0 but for compound bonds); the parameters of every term padded to B200MD_CUSTOM_MAX_PARAMS in the record,
// packed to the widest object's count when sent
struct CustomPrograms {
    vector<int> progStart = vector<int>(1, 0), op, arg; vector<double> imm;
    vector<int> exprProg, particles, periodic;
    int stride = 0;
    int numExpressions() const { return (int) exprProg.size(); }
    // the programs of one more expression
    void add(const vector<b200md_custom::Program>& programs, int numParticles, bool usesPeriodic) {
        exprProg.push_back((int) progStart.size() - 1);
        particles.push_back(numParticles);
        periodic.push_back(usesPeriodic ? 1 : 0);
        for (const b200md_custom::Program& p : programs) {
            op.insert(op.end(), p.op.begin(), p.op.end());
            arg.insert(arg.end(), p.arg.begin(), p.arg.end());
            imm.insert(imm.end(), p.imm.begin(), p.imm.end());
            progStart.push_back((int) op.size());
        }
    }
    vector<double> packed(const TermRecord& r) const {
        const size_t n = r.size();
        vector<double> p(n*stride);
        for (size_t i = 0; i < n; i++)
            for (int k = 0; k < stride; k++) p[i*stride + k] = r.params[0][i*B200MD_CUSTOM_MAX_PARAMS + k];
        return p;
    }
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
               rb{B200MD_BONDED_RB_TORSIONS, 4, 0, 1}, cmap{B200MD_BONDED_CMAP, 1, 1, 0};
    // the custom terms of each class (B200MD_CUSTOM_*): one atom column (a compound bond's B200MD_CUSTOM_MAX_PARTICLES
    // entries, unused ones -1; a centroid bond's are groups), the expression, the parameters
    TermRecord customTerms[6] = {{B200MD_BONDED_CUSTOM_TORSIONS, 1, 1, 1}, {B200MD_BONDED_CUSTOM_BONDS, 1, 1, 1},
                                 {B200MD_BONDED_CUSTOM_EXTERNALS, 1, 1, 1}, {B200MD_BONDED_CUSTOM_ANGLES, 1, 1, 1},
                                 {B200MD_BONDED_CUSTOM_COMPOUND, 1, 1, 1}, {B200MD_BONDED_CUSTOM_CENTROID, 1, 1, 1}};
    // the groups of every CustomCentroidBondForce object, one object's after the other's (a bond's group indices count from the
    // first group of all objects): CSR over atoms with the normalised weights of computeNormalizedWeights
    vector<int> centroidGroupStart = vector<int>(1, 0), centroidGroupAtoms;
    vector<double> centroidGroupWeights;
    // CMAP: the maps of all objects one after the other (a term's map index counts from the first map of all objects);
    // coefficients from CMAPTorsionForceImpl::calcMapDerivatives, [sum size^2][16]
    vector<int> cmapSize; vector<double> cmapCoeff;
    // RMSDForce objects in the order their kernels were initialised: particle lists (an empty list expanded to every particle)
    // with the reference position of each listed particle, and the force groups
    int cvCount = 0;                // collective variables of the System's CustomCVForce
    vector<vector<int> > rmsdParticles; vector<vector<double> > rmsdRef; vector<int> rmsdGroup;
    void rmsdArrays(vector<int>& start, vector<int>& atoms, vector<double>& ref) const {
        start.assign(1, 0); atoms.clear(); ref.clear();
        for (size_t o = 0; o < rmsdParticles.size(); o++) {
            atoms.insert(atoms.end(), rmsdParticles[o].begin(), rmsdParticles[o].end());
            ref.insert(ref.end(), rmsdRef[o].begin(), rmsdRef[o].end());
            start.push_back((int) atoms.size());
        }
    }
    // CustomNonbondedForce objects in the order their kernels were initialised: programs, tables, per-particle parameters
    // ([particle][P] per object), switching distance (-1: none), force group and long-range coefficient; the method, cutoff and
    // excluded pairs they share (validateSystem has checked that they do)
    CustomPrograms cnbPrograms;
    b200md_custom::Tables cnbTables;
    vector<vector<double> > cnbParams; vector<int> cnbNumParams, cnbGroup; vector<double> cnbSwitch, cnbLrc;
    int cnbMethod = 0; double cnbCutoff = 0; vector<int> cnbExcl1, cnbExcl2;
    int cnbStride() const { int s = 0; for (int p : cnbNumParams) s = max(s, p); return s; }
    // the parameters of every object as b200md_set_custom_nonbonded takes them: [object][particle][stride]
    vector<double> cnbPacked() const {
        const int stride = cnbStride();
        vector<double> p(cnbParams.size()*numParticles*stride, 0.0);
        for (size_t o = 0; o < cnbParams.size(); o++)
            for (int i = 0; i < numParticles; i++)
                for (int k = 0; k < cnbNumParams[o]; k++) p[(o*numParticles + i)*stride + k] = cnbParams[o][(size_t) i*cnbNumParams[o] + k];
        return p;
    }
    // the programs of each custom class
    CustomPrograms customPrograms[6];
    // the global parameters the expressions of all custom classes read: slot of every name (shared by all objects) and the
    // value last sent
    map<string, int> customGlobalSlot;
    vector<double> customGlobals;
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
        typedef int (*SetCustom)(b200md_ctx*, int, const int*, const int*, const int*, const double*, int, int, const int*, const int*, const double*);
        const SetCustom setCustom[4] = {b200md_set_custom_torsions, b200md_set_custom_bonds, b200md_set_custom_externals, b200md_set_custom_angles};
        for (int k = 0; k < 6; k++) {
            const TermRecord& r = customTerms[k];
            if (!r.size()) continue;
            const CustomPrograms& c = customPrograms[k];
            const vector<double> par = c.packed(r);
            if (k == B200MD_CUSTOM_CENTROID)
                check(b200md_set_custom_centroid(ctx, c.numExpressions(), c.particles.data(), c.periodic.data(), c.progStart.data(), c.op.data(),
                                                 c.arg.data(), c.imm.data(), c.stride, r.size(), r.ints[0].data(), r.atoms[0].data(), par.data(),
                                                 (int) centroidGroupStart.size() - 1, centroidGroupStart.data(), centroidGroupAtoms.data(),
                                                 centroidGroupWeights.data()));
            else if (k == B200MD_CUSTOM_COMPOUND)
                check(b200md_set_custom_compound(ctx, c.numExpressions(), c.particles.data(), c.periodic.data(), c.progStart.data(), c.op.data(),
                                                 c.arg.data(), c.imm.data(), c.stride, r.size(), r.ints[0].data(), r.atoms[0].data(), par.data()));
            else
                check(setCustom[k](ctx, c.numExpressions(), c.progStart.data(), c.op.data(), c.arg.data(), c.imm.data(), c.stride, r.size(),
                                   r.ints[0].data(), r.atoms[0].data(), par.data()));
            check(b200md_set_bonded_groups(ctx, r.kind, r.size(), r.group.data()));
        }
        if (!customGlobals.empty()) check(b200md_set_custom_globals(ctx, (int) customGlobals.size(), customGlobals.data()));
        if (!cnbGroup.empty()) {
            const CustomPrograms& c = cnbPrograms;
            const vector<double> par = cnbPacked();
            check(b200md_set_custom_nonbonded(ctx, cnbMethod, cnbCutoff, (int) cnbGroup.size(), c.progStart.data(), c.op.data(), c.arg.data(),
                                              c.imm.data(), cnbNumParams.data(), cnbStride(), par.data(), cnbSwitch.data(), cnbGroup.data(),
                                              (int) cnbExcl1.size(), cnbExcl1.data(), cnbExcl2.data()));
            check(b200md_set_custom_tables(ctx, cnbTables.count(), cnbTables.dims.data(), cnbTables.start.data(), cnbTables.values.data()));
        }
        if (!rmsdGroup.empty()) {
            vector<int> start, atoms; vector<double> ref;
            rmsdArrays(start, atoms, ref);
            check(b200md_set_rmsd(ctx, (int) rmsdGroup.size(), start.data(), atoms.data(), ref.data(), rmsdGroup.data()));
        }
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
    // changed: the message for a changed atom, if not "The set of particles in <aTerm> has changed"
    template<class Read> TermRecord reread(PlatformData& d, const TermRecord& r, int numTerms, const char* terms, const char* aTerm, Read read,
                                           const char* changed = nullptr) const {
        d.ensureFinalized();
        d.dropForces();
        if (numTerms != count) throw OpenMMException(string("updateParametersInContext: The number of ") + terms + " has changed");
        TermRecord fresh(r.kind, r.atoms.size(), r.ints.size(), r.params.size());
        for (int i = 0; i < count; i++) read(i, fresh);
        for (size_t c = 0; c < r.atoms.size(); c++)
            if (!equal(fresh.atoms[c].begin(), fresh.atoms[c].end(), start(r.atoms[c], r)))
                throw OpenMMException(string("updateParametersInContext: ") + (changed ? string(changed) : string("The set of particles in ") + aTerm + " has changed"));
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

// What the custom kernels differ in (B200CalcCustomForceKernel below): the Force, its class and term bit, the names in
// messages, how its expression is translated, its particles per term and whether its point functions take the minimum image
// (compound and centroid bonds only), how term i is read, the groups of atoms the object adds (centroid bonds only: addGroups
// returns the index its first group gets, which read adds to the object's own group indices), and the call that sends new
// parameters.  CustomTerms is what the torsion, bond, external and angle classes share: an expression of the class's
// variables, translated by translateExpression.
struct NoGroups {
    template<class F> static int addGroups(PlatformData&, const System&, const F&) { return 0; }
};
template<class T> struct CustomTerms : NoGroups {
    template<class F> static void translate(const F& force, map<string, int>& globalSlot, vector<b200md_custom::Program>& programs) {
        vector<string> params, globals;
        for (int i = 0; i < T::numParams(force); i++) params.push_back(T::paramName(force, i));
        for (int i = 0; i < force.getNumGlobalParameters(); i++) globals.push_back(force.getGlobalParameterName(i));
        b200md_custom::translateExpression(force.getEnergyFunction(), T::variables(), T::name, T::perTerm, T::cls == B200MD_CUSTOM_EXTERNAL,
                                           params, globals, globalSlot, programs);
    }
    template<class F> static int particles(const F&) { return 0; }
    template<class F> static bool periodic(const F&) { return false; }
};
struct CustomTorsions : CustomTerms<CustomTorsions> {
    typedef CustomTorsionForce Force; typedef CalcCustomTorsionForceKernel Kernel;
    enum { cls = B200MD_CUSTOM_TORSION, bit = B200MD_TERM_CUSTOM_TORSIONS };
    static constexpr const char* name = "CustomTorsionForce", *terms = "torsions", *aTerm = "a torsion", *perTerm = "torsion", *changed = nullptr;
    static vector<string> variables() { return {"theta"}; }
    static int count(const Force& f) { return f.getNumTorsions(); }
    static int numParams(const Force& f) { return f.getNumPerTorsionParameters(); }
    static string paramName(const Force& f, int i) { return f.getPerTorsionParameterName(i); }
    static vector<int> read(const Force& f, int i, vector<double>& par, int) { int a, b, c, e; f.getTorsionParameters(i, a, b, c, e, par); return {a, b, c, e}; }
    static int update(b200md_ctx* c, int n, const double* p) { return b200md_update_custom_torsion_params(c, n, p); }
    static int numParamDerivatives(const Force& f) { return f.getNumEnergyParameterDerivatives(); }
};
struct CustomBonds : CustomTerms<CustomBonds> {
    typedef CustomBondForce Force; typedef CalcCustomBondForceKernel Kernel;
    enum { cls = B200MD_CUSTOM_BOND, bit = B200MD_TERM_CUSTOM_BONDS };
    static constexpr const char* name = "CustomBondForce", *terms = "bonds", *aTerm = "a bond", *perTerm = "bond", *changed = nullptr;
    static vector<string> variables() { return {"r"}; }
    static int count(const Force& f) { return f.getNumBonds(); }
    static int numParams(const Force& f) { return f.getNumPerBondParameters(); }
    static string paramName(const Force& f, int i) { return f.getPerBondParameterName(i); }
    static vector<int> read(const Force& f, int i, vector<double>& par, int) { int a, b; f.getBondParameters(i, a, b, par); return {a, b}; }
    static int update(b200md_ctx* c, int n, const double* p) { return b200md_update_custom_bond_params(c, n, p); }
    static int numParamDerivatives(const Force& f) { return f.getNumEnergyParameterDerivatives(); }
};
struct CustomExternals : CustomTerms<CustomExternals> {
    typedef CustomExternalForce Force; typedef CalcCustomExternalForceKernel Kernel;
    enum { cls = B200MD_CUSTOM_EXTERNAL, bit = B200MD_TERM_CUSTOM_EXTERNALS };
    static constexpr const char* name = "CustomExternalForce", *terms = "particles", *aTerm = "a particle", *perTerm = "particle",
                                 *changed = "A particle index has changed";
    static vector<string> variables() { return {"x", "y", "z"}; }
    static int count(const Force& f) { return f.getNumParticles(); }
    static int numParams(const Force& f) { return f.getNumPerParticleParameters(); }
    static string paramName(const Force& f, int i) { return f.getPerParticleParameterName(i); }
    static vector<int> read(const Force& f, int i, vector<double>& par, int) { int a; f.getParticleParameters(i, a, par); return {a}; }
    static int update(b200md_ctx* c, int n, const double* p) { return b200md_update_custom_external_params(c, n, p); }
    static int numParamDerivatives(const Force&) { return 0; }        // CustomExternalForce has none
};
struct CustomAngles : CustomTerms<CustomAngles> {
    typedef CustomAngleForce Force; typedef CalcCustomAngleForceKernel Kernel;
    enum { cls = B200MD_CUSTOM_ANGLE, bit = B200MD_TERM_CUSTOM_ANGLES };
    static constexpr const char* name = "CustomAngleForce", *terms = "angles", *aTerm = "an angle", *perTerm = "angle", *changed = nullptr;
    static vector<string> variables() { return {"theta"}; }
    static int count(const Force& f) { return f.getNumAngles(); }
    static int numParams(const Force& f) { return f.getNumPerAngleParameters(); }
    static string paramName(const Force& f, int i) { return f.getPerAngleParameterName(i); }
    static vector<int> read(const Force& f, int i, vector<double>& par, int) { int a, b, c; f.getAngleParameters(i, a, b, c, par); return {a, b, c}; }
    static int update(b200md_ctx* c, int n, const double* p) { return b200md_update_custom_angle_params(c, n, p); }
    static int numParamDerivatives(const Force& f) { return f.getNumEnergyParameterDerivatives(); }
};
// A compound bond's expression is of the coordinates of its particles: 1 + 3 (particles per bond) programs, which k_compound
// interprets.  Its atoms are padded to B200MD_CUSTOM_MAX_PARTICLES with -1.
struct CustomCompounds : NoGroups {
    typedef CustomCompoundBondForce Force; typedef CalcCustomCompoundBondForceKernel Kernel;
    enum { cls = B200MD_CUSTOM_COMPOUND, bit = B200MD_TERM_CUSTOM_COMPOUND };
    static constexpr const char* name = "CustomCompoundBondForce", *terms = "bonds", *aTerm = "a bond", *changed = nullptr;
    static int count(const Force& f) { return f.getNumBonds(); }
    static int numParams(const Force& f) { return f.getNumPerBondParameters(); }
    static vector<int> read(const Force& f, int i, vector<double>& par, int) {
        vector<int> atoms;
        f.getBondParameters(i, atoms, par);
        atoms.resize(B200MD_CUSTOM_MAX_PARTICLES, -1);
        return atoms;
    }
    static int update(b200md_ctx* c, int n, const double* p) { return b200md_update_custom_compound_params(c, n, p); }
    static int numParamDerivatives(const Force& f) { return f.getNumEnergyParameterDerivatives(); }
    static void translate(const Force& f, map<string, int>& globalSlot, vector<b200md_custom::Program>& programs) {
        b200md_custom::translateCompound(f, globalSlot, programs);
    }
    static int particles(const Force& f) { return f.getNumParticlesPerBond(); }
    static bool periodic(const Force& f) { return f.usesPeriodicBoundaryConditions(); }
};
// A centroid bond's expression is a compound bond's of the centres of its groups: the same programs, which k_compound runs at
// the centres k_centroid_centers makes.  Its groups are padded to B200MD_CUSTOM_MAX_PARTICLES with -1, and its objects' groups
// go into one table, with the weights CustomCentroidBondForceImpl::computeNormalizedWeights makes (masses by default; a
// group whose weights add to 0 raises the reference's error there).
struct CustomCentroids {
    typedef CustomCentroidBondForce Force; typedef CalcCustomCentroidBondForceKernel Kernel;
    enum { cls = B200MD_CUSTOM_CENTROID, bit = B200MD_TERM_CUSTOM_CENTROID };
    static constexpr const char* name = "CustomCentroidBondForce", *terms = "bonds", *aTerm = "a bond",
                                 *changed = "The set of groups in a bond has changed";
    static int count(const Force& f) { return f.getNumBonds(); }
    static int numParams(const Force& f) { return f.getNumPerBondParameters(); }
    static vector<int> read(const Force& f, int i, vector<double>& par, int base) {
        vector<int> groups;
        f.getBondParameters(i, groups, par);
        for (int& g : groups) g += base;
        groups.resize(B200MD_CUSTOM_MAX_PARTICLES, -1);
        return groups;
    }
    static int update(b200md_ctx* c, int n, const double* p) { return b200md_update_custom_centroid_params(c, n, p); }
    static int numParamDerivatives(const Force& f) { return f.getNumEnergyParameterDerivatives(); }
    static void translate(const Force& f, map<string, int>& globalSlot, vector<b200md_custom::Program>& programs) {
        b200md_custom::translateCentroid(f, globalSlot, programs);
    }
    static int particles(const Force& f) { return f.getNumGroupsPerBond(); }
    static bool periodic(const Force& f) { return f.usesPeriodicBoundaryConditions(); }
    static int addGroups(PlatformData& d, const System& system, const Force& f) {
        const int base = (int) d.centroidGroupStart.size() - 1;
        vector<vector<double> > weights;
        CustomCentroidBondForceImpl::computeNormalizedWeights(f, system, weights);
        for (int g = 0; g < f.getNumGroups(); g++) {
            vector<int> atoms;
            vector<double> given;
            f.getGroupParameters(g, atoms, given);
            d.centroidGroupAtoms.insert(d.centroidGroupAtoms.end(), atoms.begin(), atoms.end());
            d.centroidGroupWeights.insert(d.centroidGroupWeights.end(), weights[g].begin(), weights[g].end());
            d.centroidGroupStart.push_back((int) d.centroidGroupAtoms.size());
        }
        return base;
    }
};

// The global parameters one custom force object's expression reads, and their slots in the Context's shared map
struct ObjectGlobals {
    vector<pair<string, int> > slots;
    // after the object's expression was translated.  The Context's parameter map does not exist yet (ContextImpl.cpp:120-131
    // fills it after the kernels are initialised): start from the defaults, send() sends whatever differs
    template<class F> void init(PlatformData& d, const F& force) {
        d.customGlobals.resize(d.customGlobalSlot.size(), 0.0);
        for (int i = 0; i < force.getNumGlobalParameters(); i++) {
            const map<string, int>::const_iterator it = d.customGlobalSlot.find(force.getGlobalParameterName(i));
            if (it == d.customGlobalSlot.end()) continue;         // declared, but the expression does not read it
            slots.push_back(make_pair(it->first, it->second));
            d.customGlobals[it->second] = force.getGlobalParameterDefaultValue(i);
        }
    }
    // execute: a changed global value is a stream-ordered copy into the buffer the step graph reads (NonbondedForce offsets alike)
    void send(PlatformData& d, ContextImpl& context) const {
        bool changed = false;
        for (const pair<string, int>& s : slots) {
            const double v = context.getParameter(s.first);
            if (v != d.customGlobals[s.second]) { d.customGlobals[s.second] = v; changed = true; }
        }
        if (changed) d.check(b200md_set_custom_globals(d.ctx, (int) d.customGlobals.size(), d.customGlobals.data()));
    }
};

// CustomTorsionForce, CustomBondForce, CustomExternalForce, CustomAngleForce, CustomCompoundBondForce and
// CustomCentroidBondForce (T: CustomTorsions, CustomBonds, CustomExternals, CustomAngles, CustomCompounds, CustomCentroids):
// the expression becomes 1 + (number of variables) instruction programs, which k_custom interprets (k_compound for compound
// and centroid bonds).
template<class T>
class B200CalcCustomForceKernel : public T::Kernel, ObjectTerms {
public:
    B200CalcCustomForceKernel(string name, const Platform& platform, ContextImpl& context) : T::Kernel(name, platform), context(context) {}
    // the term's parameters: as many as the force declares (the Reference platform reads as many), padded with zeros
    void read(const typename T::Force& force, int i, TermRecord& r) const {
        vector<double> par;
        const vector<int> atoms = T::read(force, i, par, groupBase);
        par.resize(numParams);
        par.resize(B200MD_CUSTOM_MAX_PARAMS, 0.0);
        r.add(atoms, {expr}, par);
    }
    void initialize(const System& system, const typename T::Force& force) {
        PlatformData& d = getData(context);
        CustomPrograms& c = d.customPrograms[T::cls];
        expr = c.numExpressions();
        numParams = T::numParams(force);
        if (d.finalized) throw OpenMMException(string("B200 platform: ") + T::name + " initialised after the Context was finalised");
        groupBase = T::addGroups(d, system, force);
        add(d, d.customTerms[T::cls], force, T::count(force), T::bit, T::name, [&](int i, TermRecord& r) { read(force, i, r); });
        vector<b200md_custom::Program> programs;
        T::translate(force, d.customGlobalSlot, programs);
        c.add(programs, T::particles(force), T::periodic(force));
        globals.init(d, force);
        c.stride = max(c.stride, numParams);
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) {
        PlatformData& d = getData(context);
        globals.send(d, context);
        d.pendingTerms |= T::bit;
        return 0.0;
    }
    void copyParametersToContext(ContextImpl& context, const typename T::Force& force) {
        PlatformData& d = getData(context);
        TermRecord& r = d.customTerms[T::cls];
        store(r, reread(d, r, T::count(force), T::terms, T::aTerm, [&](int i, TermRecord& f) { read(force, i, f); }, T::changed));
        const vector<double> packed = d.customPrograms[T::cls].packed(r);
        d.check(T::update(d.ctx, r.size(), packed.data()));
    }
private:
    ContextImpl& context;
    int expr = 0, numParams = 0;          // this object's expression; its number of per-term parameters
    int groupBase = 0;                    // the index of this object's first group (centroid bonds)
    ObjectGlobals globals;
};

// GBSAOBCForce: the per-atom parameters go to the engine at initialize; execute() only records the term, so the lazy fused
// step covers it like every other force.  validateSystem has checked the method against the NonbondedForce's.
class B200CalcGBSAOBCForceKernel : public CalcGBSAOBCForceKernel {
public:
    B200CalcGBSAOBCForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcGBSAOBCForceKernel(name, platform), context(context) {}
    static void read(const GBSAOBCForce& force, vector<double>& q, vector<double>& r, vector<double>& s) {
        const int n = force.getNumParticles();
        q.resize(n); r.resize(n); s.resize(n);
        for (int i = 0; i < n; i++) force.getParticleParameters(i, q[i], r[i], s[i]);
    }
    void initialize(const System& system, const GBSAOBCForce& force) {
        PlatformData& d = getData(context);
        if (d.finalized) throw OpenMMException("B200 platform: GBSAOBCForce initialised after the Context was finalised");
        vector<double> q, r, s;
        read(force, q, r, s);
        const int method = force.getNonbondedMethod() == GBSAOBCForce::NoCutoff ? B200MD_NB_NOCUTOFF :
                           force.getNonbondedMethod() == GBSAOBCForce::CutoffNonPeriodic ? B200MD_NB_CUTOFF_NONPERIODIC : B200MD_NB_CUTOFF_PERIODIC;
        d.check(b200md_set_gbsa(d.ctx, method, force.getCutoffDistance(), force.getSoluteDielectric(), force.getSolventDielectric(),
                                force.getSurfaceAreaEnergy(), q.data(), r.data(), s.data()));
        d.systemTerms |= B200MD_TERM_GBSA;
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) { getData(context).pendingTerms |= B200MD_TERM_GBSA; return 0.0; }
    void copyParametersToContext(ContextImpl& context, const GBSAOBCForce& force) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        if (force.getNumParticles() != d.numParticles) throw OpenMMException("updateParametersInContext: The number of particles has changed");
        vector<double> q, r, s;
        read(force, q, r, s);
        d.check(b200md_update_gbsa_params(d.ctx, (int) q.size(), q.data(), r.data(), s.data()));
    }
private:
    ContextImpl& context;
};

// RMSDForce: the particle list and reference positions go to the engine at finalize, with those of every other RMSDForce;
// execute() only records the term, so the step graph covers it.  RMSDForceImpl has checked the particle indices and the
// number of reference positions.
class B200CalcRMSDForceKernel : public CalcRMSDForceKernel {
public:
    B200CalcRMSDForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcRMSDForceKernel(name, platform), context(context) {}
    // the particle list (empty: every particle, as ReferenceCalcRMSDForceKernel) and the reference position of each
    static void read(const RMSDForce& force, int numParticles, vector<int>& particles, vector<double>& ref) {
        particles = force.getParticles();
        if (particles.empty())
            for (int i = 0; i < numParticles; i++) particles.push_back(i);
        const vector<Vec3>& pos = force.getReferencePositions();
        ref.clear();
        for (int i : particles) for (int k = 0; k < 3; k++) ref.push_back(pos[i][k]);
    }
    void initialize(const System& system, const RMSDForce& force) {
        PlatformData& d = getData(context);
        if (d.finalized) throw OpenMMException("B200 platform: RMSDForce initialised after the Context was finalised");
        index = (int) d.rmsdGroup.size();
        numReference = (int) force.getReferencePositions().size();
        d.rmsdParticles.emplace_back(); d.rmsdRef.emplace_back();
        read(force, system.getNumParticles(), d.rmsdParticles.back(), d.rmsdRef.back());
        d.rmsdGroup.push_back(force.getForceGroup());
        d.systemTerms |= B200MD_TERM_RMSD; d.bondedGroupsUsed |= 1u << force.getForceGroup();
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) { getData(context).pendingTerms |= B200MD_TERM_RMSD; return 0.0; }
    void copyParametersToContext(ContextImpl& context, const RMSDForce& force) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        if ((int) force.getReferencePositions().size() != numReference)
            throw OpenMMException("updateParametersInContext: The number of reference positions has changed");
        read(force, d.numParticles, d.rmsdParticles[index], d.rmsdRef[index]);
        vector<int> start, atoms; vector<double> ref;
        d.rmsdArrays(start, atoms, ref);
        d.check(b200md_update_rmsd(d.ctx, (int) d.rmsdGroup.size(), start.data(), atoms.data(), ref.data()));
    }
private:
    ContextImpl& context;
    int index = 0, numReference = 0;
};

// CustomNonbondedForce: the programs, tables, parameters and exclusions go to the engine at finalize, with those of every other
// CustomNonbondedForce; execute() only records the term, so the step graph covers it.  The long-range correction is computed
// on the host as ReferenceCalcCustomNonbondedForceKernel does (CutoffPeriodic only): at the first evaluation, again when a
// global parameter the force declares changes and at copyParametersToContext; the engine adds coefficient/volume.
class B200CalcCustomNonbondedForceKernel : public CalcCustomNonbondedForceKernel {
public:
    B200CalcCustomNonbondedForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcCustomNonbondedForceKernel(name, platform), context(context) {}
    ~B200CalcCustomNonbondedForceKernel() { delete forceCopy; }
    static void read(const CustomNonbondedForce& force, vector<double>& params) {
        const int n = force.getNumParticles(), np = force.getNumPerParticleParameters();
        params.assign((size_t) n*np, 0.0);
        vector<double> p;
        for (int i = 0; i < n; i++) {
            force.getParticleParameters(i, p);
            for (int k = 0; k < np && k < (int) p.size(); k++) params[(size_t) i*np + k] = p[k];
        }
    }
    void initialize(const System& system, const CustomNonbondedForce& force) {
        PlatformData& d = getData(context);
        if (d.finalized) throw OpenMMException("B200 platform: CustomNonbondedForce initialised after the Context was finalised");
        if (force.getNumParticles() != system.getNumParticles())
            throw OpenMMException("CustomNonbondedForce must have exactly as many particles as the System it belongs to.");
        index = (int) d.cnbGroup.size();
        vector<b200md_custom::Program> programs;
        b200md_custom::translateNonbonded(force, d.customGlobalSlot, programs, d.cnbTables);
        d.cnbPrograms.add(programs, 0, false);
        globals.init(d, force);
        d.cnbParams.emplace_back();
        read(force, d.cnbParams.back());
        d.cnbNumParams.push_back(force.getNumPerParticleParameters());
        const CustomNonbondedForce::NonbondedMethod m = force.getNonbondedMethod();
        d.cnbMethod = m == CustomNonbondedForce::NoCutoff ? B200MD_NB_NOCUTOFF : m == CustomNonbondedForce::CutoffNonPeriodic ?
                      B200MD_NB_CUTOFF_NONPERIODIC : B200MD_NB_CUTOFF_PERIODIC;
        d.cnbCutoff = force.getCutoffDistance();
        d.cnbSwitch.push_back(m != CustomNonbondedForce::NoCutoff && force.getUseSwitchingFunction() ? force.getSwitchingDistance() : -1.0);
        d.cnbGroup.push_back(force.getForceGroup());
        d.cnbLrc.push_back(0.0);
        if (index == 0)
            for (int k = 0; k < force.getNumExclusions(); k++) {
                int a, b;
                force.getExclusionParticles(k, a, b);
                d.cnbExcl1.push_back(a); d.cnbExcl2.push_back(b);
            }
        if (m == CustomNonbondedForce::CutoffPeriodic && force.getUseLongRangeCorrection()) {
            forceCopy = new CustomNonbondedForce(force);
            lrcPending = true;
        }
        for (int i = 0; i < force.getNumGlobalParameters(); i++) {
            globalNames.push_back(force.getGlobalParameterName(i));
            globalValues.push_back(force.getGlobalParameterDefaultValue(i));
        }
        d.systemTerms |= B200MD_TERM_CUSTOM_NONBONDED; d.bondedGroupsUsed |= 1u << force.getForceGroup();
    }
    double execute(ContextImpl& context, bool includeForces, bool includeEnergy) {
        PlatformData& d = getData(context);
        globals.send(d, context);
        for (size_t i = 0; i < globalNames.size(); i++) {
            const double v = context.getParameter(globalNames[i]);
            if (v != globalValues[i]) { globalValues[i] = v; lrcPending = lrcPending || forceCopy != nullptr; }
        }
        if (lrcPending) sendLongRangeCorrection(d, context);
        d.pendingTerms |= B200MD_TERM_CUSTOM_NONBONDED;
        return 0.0;
    }
    void copyParametersToContext(ContextImpl& context, const CustomNonbondedForce& force) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        d.dropForces();
        if (force.getNumParticles() != d.numParticles) throw OpenMMException("updateParametersInContext: The number of particles has changed");
        if (force.getNumPerParticleParameters() != d.cnbNumParams[index])
            throw OpenMMException("updateParametersInContext: The number of per-particle parameters has changed");
        read(force, d.cnbParams[index]);
        const vector<double> par = d.cnbPacked();
        d.check(b200md_update_custom_nonbonded_params(d.ctx, d.numParticles, par.data()));
        if (forceCopy != nullptr) {
            // a new deep copy: CustomNonbondedForce's assignment would share the tabulated functions, which both then delete
            delete forceCopy;
            forceCopy = new CustomNonbondedForce(force);
            sendLongRangeCorrection(d, context);
        }
    }
private:
    // CustomNonbondedForceImpl::calcLongRangeCorrection at the Context's current global parameter values
    void sendLongRangeCorrection(PlatformData& d, ContextImpl& context) {
        vector<double> derivatives;
        CustomNonbondedForceImpl::calcLongRangeCorrection(*forceCopy, context.getOwner(), d.cnbLrc[index], derivatives);
        lrcPending = false;
        d.check(b200md_set_custom_nonbonded_lrc(d.ctx, (int) d.cnbLrc.size(), d.cnbLrc.data()));
    }
    ContextImpl& context;
    int index = 0;                                  // this object among the Context's CustomNonbondedForce objects
    CustomNonbondedForce* forceCopy = nullptr;      // for the long-range correction (CutoffPeriodic with it on)
    bool lrcPending = false;
    vector<string> globalNames; vector<double> globalValues;
    ObjectGlobals globals;
};

// CustomCVForce: CustomCVForceImpl (the reference's, untouched) builds an inner System of the collective variables, one force
// group each, and a linked Context on this platform, so the inner Context is an ordinary engine on the same device.  execute()
// copies the state to it on the device, evaluates each variable's group there and snapshots its forces into the outer
// context's slot, evaluates the energy expression and its derivatives on the host with Lepton (one host sync per variable, as
// on the reference's GPU platforms), uploads dE/dCV_i and records the term: the forces are combined inside the outer
// evaluation, the fused step graph included.
class B200CalcCustomCVForceKernel : public CalcCustomCVForceKernel {
public:
    B200CalcCustomCVForceKernel(string name, const Platform& platform, ContextImpl& context) : CalcCustomCVForceKernel(name, platform), context(context) {}
    void initialize(const System& system, const CustomCVForce& force, ContextImpl& innerContext) {
        PlatformData& d = getData(context);
        if (d.finalized) throw OpenMMException("B200 platform: CustomCVForce initialised after the Context was finalised");
        if (d.cvCount) throw OpenMMException("B200 platform: only one CustomCVForce per System is supported");
        if (force.getNumEnergyParameterDerivatives() > 0) throw OpenMMException("B200 platform: energy parameter derivatives of a CustomCVForce are not supported");
        for (int i = 0; i < force.getNumCollectiveVariables(); i++) variableNames.push_back(force.getCollectiveVariableName(i));
        for (int i = 0; i < force.getNumGlobalParameters(); i++) globalNames.push_back(force.getGlobalParameterName(i));
        build(force);
        d.cvCount = (int) variableNames.size();
        d.check(b200md_set_cv_forces(d.ctx, d.cvCount));
        d.systemTerms |= B200MD_TERM_CV_FORCES;
    }
    double execute(ContextImpl& context, ContextImpl& innerContext, bool includeForces, bool includeEnergy) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        copyState(context, innerContext);
        PlatformData& inner = getData(innerContext);
        map<string, double> variables;
        for (const string& name : globalNames) variables[name] = context.getParameter(name);
        const int n = (int) variableNames.size();
        for (int i = 0; i < n; i++) {
            variables[variableNames[i]] = innerContext.calcForcesAndEnergy(true, true, 1 << i);
            if (includeForces) d.check(b200md_cv_snapshot_forces(inner.ctx, d.ctx, i));
        }
        if (includeForces) {
            vector<double> coeff(n);
            for (int i = 0; i < n; i++) coeff[i] = derivs[i].evaluate(variables);
            d.check(b200md_set_cv_coefficients(d.ctx, n, coeff.data()));
            d.pendingTerms |= B200MD_TERM_CV_FORCES;
        }
        return includeEnergy ? energy.evaluate(variables) : 0.0;
    }
    // the positions, box and global parameters of the outer Context into the inner one (getCollectiveVariableValues reads it)
    void copyState(ContextImpl& context, ContextImpl& innerContext) {
        PlatformData& d = getData(context);
        d.ensureFinalized();
        PlatformData& inner = getData(innerContext);
        inner.ensureFinalized();
        inner.dropForces();
        for (auto& p : innerContext.getParameters()) innerContext.setParameter(p.first, context.getParameter(p.first));
        if (b200md_cv_copy_state(d.ctx, inner.ctx) != 0) d.check(-1);
        inner.boxError = d.boxError;
    }
    void copyParametersToContext(ContextImpl& context, const CustomCVForce& force) { build(force); }
private:
    // the energy expression and its derivatives by the variables, with the force's tabulated functions as the Reference
    // platform's splines (ReferenceCustomCVForce)
    void build(const CustomCVForce& force) {
        map<string, Lepton::CustomFunction*> functions;
        for (int i = 0; i < force.getNumTabulatedFunctions(); i++)
            functions[force.getTabulatedFunctionName(i)] = createReferenceTabulatedFunction(force.getTabulatedFunction(i));
        try {
            Lepton::ParsedExpression expr = Lepton::Parser::parse(force.getEnergyFunction(), functions);
            energy = expr.createProgram();
            derivs.clear();
            for (const string& name : variableNames) derivs.push_back(expr.differentiate(name).optimize().createProgram());
        } catch (...) {
            for (auto& f : functions) delete f.second;
            throw;
        }
        for (auto& f : functions) delete f.second;
    }
    ContextImpl& context;
    vector<string> variableNames, globalNames;
    Lepton::ExpressionProgram energy;
    vector<Lepton::ExpressionProgram> derivs;
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
        if (name == CalcCustomTorsionForceKernel::Name()) return new B200CalcCustomForceKernel<CustomTorsions>(name, platform, context);
        if (name == CalcCustomBondForceKernel::Name()) return new B200CalcCustomForceKernel<CustomBonds>(name, platform, context);
        if (name == CalcCustomExternalForceKernel::Name()) return new B200CalcCustomForceKernel<CustomExternals>(name, platform, context);
        if (name == CalcCustomAngleForceKernel::Name()) return new B200CalcCustomForceKernel<CustomAngles>(name, platform, context);
        if (name == CalcCustomCompoundBondForceKernel::Name()) return new B200CalcCustomForceKernel<CustomCompounds>(name, platform, context);
        if (name == CalcCustomCentroidBondForceKernel::Name()) return new B200CalcCustomForceKernel<CustomCentroids>(name, platform, context);
        if (name == CalcGBSAOBCForceKernel::Name()) return new B200CalcGBSAOBCForceKernel(name, platform, context);
        if (name == CalcRMSDForceKernel::Name()) return new B200CalcRMSDForceKernel(name, platform, context);
        if (name == CalcCustomNonbondedForceKernel::Name()) return new B200CalcCustomNonbondedForceKernel(name, platform, context);
        if (name == CalcCustomCVForceKernel::Name()) return new B200CalcCustomCVForceKernel(name, platform, context);
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
                                CalcCustomTorsionForceKernel::Name(), CalcCustomBondForceKernel::Name(), CalcCustomExternalForceKernel::Name(),
                                CalcCustomAngleForceKernel::Name(), CalcCustomCompoundBondForceKernel::Name(), CalcCustomCentroidBondForceKernel::Name(),
                                CalcGBSAOBCForceKernel::Name(), CalcRMSDForceKernel::Name(), CalcCustomCVForceKernel::Name(), CalcCustomNonbondedForceKernel::Name(),
                                RemoveCMMotionKernel::Name(), IntegrateVerletStepKernel::Name(),
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
    // A custom force: getEnergyParameterDerivatives returns nothing here; an expression beyond the interpreter's limits or with
    // a tabulated function is refused; an unknown variable is an error on every platform and is raised by the kernel's
    // initialize, as the Reference platform does
    template<class T> static void validateCustom(const typename T::Force& force) {
        if (T::numParamDerivatives(force) > 0)
            throw OpenMMException(string("B200 platform: energy parameter derivatives of a ") + T::name + " are not supported");
        map<string, int> slots;
        vector<b200md_custom::Program> programs;
        try { T::translate(force, slots, programs); }
        catch (const b200md_custom::Unsupported&) { throw; }
        catch (const OpenMMException&) {}
    }
    // A GBSAOBCForce: the generalized Born chain walks the NonbondedForce's neighbour list, so its method and cutoff must be
    // that list's (CutoffPeriodic goes with CutoffPeriodic or PME, which is what ForceField builds for PME); without a
    // NonbondedForce only NoCutoff, over the list of all pairs.  Radii at or below the dielectric offset are refused too.
    static void validateGBSA(const System& system, const GBSAOBCForce& gbsa, const NonbondedForce* nonbonded) {
        if (gbsa.getNumParticles() != system.getNumParticles())
            throw OpenMMException("B200 platform: a GBSAOBCForce must have exactly as many particles as the System");
        const GBSAOBCForce::NonbondedMethod m = gbsa.getNonbondedMethod();
        if (!nonbonded) {
            if (m != GBSAOBCForce::NoCutoff) throw OpenMMException("B200 platform: a GBSAOBCForce with a cutoff needs a NonbondedForce with the same cutoff");
        }
        else {
            const NonbondedForce::NonbondedMethod n = nonbonded->getNonbondedMethod();
            const bool match = m == GBSAOBCForce::NoCutoff ? n == NonbondedForce::NoCutoff :
                               m == GBSAOBCForce::CutoffNonPeriodic ? n == NonbondedForce::CutoffNonPeriodic :
                               (n == NonbondedForce::CutoffPeriodic || n == NonbondedForce::PME);
            if (!match) throw OpenMMException("B200 platform: the GBSAOBCForce's nonbonded method does not match the NonbondedForce's");
            if (m != GBSAOBCForce::NoCutoff && gbsa.getCutoffDistance() != nonbonded->getCutoffDistance())
                throw OpenMMException("B200 platform: the GBSAOBCForce's cutoff differs from the NonbondedForce's");
        }
        for (int i = 0; i < gbsa.getNumParticles(); i++) {
            double q, r, s;
            gbsa.getParticleParameters(i, q, r, s);
            if (!(r > 0.009)) throw OpenMMException("B200 platform: a GBSAOBCForce radius at or below the dielectric offset (0.009 nm)");
        }
    }
    // A CustomNonbondedForce on its own: interaction groups, energy parameter derivatives, continuous tables, more than 8
    // per-particle parameters and programs beyond the interpreter's limits are refused (an unknown variable is left to the
    // kernel's initialize, as for the other custom forces)
    static void validateCustomNonbonded(const System& system, const CustomNonbondedForce& force) {
        if (force.getNumInteractionGroups() > 0) throw OpenMMException("B200 platform: interaction groups of a CustomNonbondedForce are not supported");
        if (force.getNumEnergyParameterDerivatives() > 0)
            throw OpenMMException("B200 platform: energy parameter derivatives of a CustomNonbondedForce are not supported");
        if (force.getNumParticles() != system.getNumParticles())
            throw OpenMMException("CustomNonbondedForce must have exactly as many particles as the System it belongs to.");
        map<string, int> slots;
        vector<b200md_custom::Program> programs;
        b200md_custom::Tables tables;
        try { b200md_custom::translateNonbonded(force, slots, programs, tables); }
        catch (const b200md_custom::Unsupported&) { throw; }
        catch (const OpenMMException&) {}
    }
    // the excluded pairs of a CustomNonbondedForce, or the exception pairs of a NonbondedForce, as a set
    static set<pair<int, int> > pairSet(const CustomNonbondedForce* c, const NonbondedForce* n) {
        set<pair<int, int> > s;
        const int count = c ? c->getNumExclusions() : n->getNumExceptions();
        for (int k = 0; k < count; k++) {
            int a, b;
            double q, sig, eps;
            if (c) c->getExclusionParticles(k, a, b);
            else n->getExceptionParameters(k, a, b, q, sig, eps);
            s.insert(make_pair(min(a, b), max(a, b)));
        }
        return s;
    }
    // The CustomNonbondedForce objects together: the pair kernel walks one neighbour list, so they share one method, one cutoff
    // and one exclusion set, and with a NonbondedForce those are its method (CutoffPeriodic with CutoffPeriodic or PME), its
    // cutoff and its exception pairs, from which the list's masks are built.  Without one the list is built at the custom
    // force's method and cutoff, which a GBSAOBCForce (at NoCutoff) can share only at NoCutoff.
    static void validateCustomNonbondedSet(const vector<const CustomNonbondedForce*>& forces, const NonbondedForce* nonbonded,
                                           const GBSAOBCForce* gbsa) {
        const CustomNonbondedForce& first = *forces[0];
        const CustomNonbondedForce::NonbondedMethod m = first.getNonbondedMethod();
        const set<pair<int, int> > excl = pairSet(&first, nullptr);
        for (const CustomNonbondedForce* f : forces) {
            if (f->getNonbondedMethod() != m || (m != CustomNonbondedForce::NoCutoff && f->getCutoffDistance() != first.getCutoffDistance()))
                throw OpenMMException("B200 platform: CustomNonbondedForce objects with different methods or cutoffs are not supported");
            if (f != &first && pairSet(f, nullptr) != excl)
                throw OpenMMException("B200 platform: CustomNonbondedForce objects with different exclusions are not supported");
        }
        if (!nonbonded) {
            // the list is then the custom force's own; a GBSAOBCForce (NoCutoff here, validateGBSA) needs every pair in it
            if (gbsa && m != CustomNonbondedForce::NoCutoff)
                throw OpenMMException("B200 platform: a GBSAOBCForce beside a CustomNonbondedForce with a cutoff needs a NonbondedForce");
            return;
        }
        const NonbondedForce::NonbondedMethod n = nonbonded->getNonbondedMethod();
        const bool match = m == CustomNonbondedForce::NoCutoff ? n == NonbondedForce::NoCutoff :
                           m == CustomNonbondedForce::CutoffNonPeriodic ? n == NonbondedForce::CutoffNonPeriodic :
                           (n == NonbondedForce::CutoffPeriodic || n == NonbondedForce::PME);
        if (!match) throw OpenMMException("B200 platform: the CustomNonbondedForce's nonbonded method does not match the NonbondedForce's");
        if (m != CustomNonbondedForce::NoCutoff && first.getCutoffDistance() != nonbonded->getCutoffDistance())
            throw OpenMMException("B200 platform: the CustomNonbondedForce's cutoff differs from the NonbondedForce's");
        if (excl != pairSet(nullptr, nonbonded))
            throw OpenMMException("B200 platform: the CustomNonbondedForce's exclusions differ from the NonbondedForce's exceptions");
    }
    // the Force classes this platform has a kernel for; a CustomCVForce's variables must be among them, since its inner
    // Context is created on this platform explicitly and cannot fall back on its own
    static bool hasKernel(const Force& f) {
        return dynamic_cast<const NonbondedForce*>(&f) || dynamic_cast<const HarmonicBondForce*>(&f) || dynamic_cast<const HarmonicAngleForce*>(&f) ||
               dynamic_cast<const PeriodicTorsionForce*>(&f) || dynamic_cast<const RBTorsionForce*>(&f) || dynamic_cast<const CMAPTorsionForce*>(&f) ||
               dynamic_cast<const CustomTorsionForce*>(&f) || dynamic_cast<const CustomBondForce*>(&f) || dynamic_cast<const CustomExternalForce*>(&f) ||
               dynamic_cast<const CustomAngleForce*>(&f) || dynamic_cast<const CustomCompoundBondForce*>(&f) ||
               dynamic_cast<const CustomCentroidBondForce*>(&f) || dynamic_cast<const GBSAOBCForce*>(&f) || dynamic_cast<const RMSDForce*>(&f) ||
               dynamic_cast<const CustomCVForce*>(&f);
    }
    // The checks of one System's forces: the System's own, or the collective variables of a CustomCVForce, which become the
    // forces of its inner System (same particles, one force group per variable), checked the same way, recursively
    static void validateForces(const System& system, const vector<const Force*>& forces) {
        int numNonbonded = 0;
        const NonbondedForce* nonbonded = nullptr;
        const GBSAOBCForce* gbsa = nullptr;
        vector<const CustomNonbondedForce*> customNonbonded;
        for (const Force* fp : forces) {
            const Force& force = *fp;
            if (const CustomCVForce* cv = dynamic_cast<const CustomCVForce*>(&force)) {
                if (cv->getNumEnergyParameterDerivatives() > 0)
                    throw OpenMMException("B200 platform: energy parameter derivatives of a CustomCVForce are not supported");
                if (cv->getNumCollectiveVariables() > 31) throw OpenMMException("B200 platform: a CustomCVForce has more than 31 collective variables");
                vector<const Force*> variables;
                for (int i = 0; i < cv->getNumCollectiveVariables(); i++) {
                    const Force& v = cv->getCollectiveVariable(i);
                    if (!hasKernel(v)) throw OpenMMException("B200 platform: a collective variable of a CustomCVForce is of a Force class this platform does not run");
                    variables.push_back(&v);
                }
                validateForces(system, variables);
            }
            if (const GBSAOBCForce* g = dynamic_cast<const GBSAOBCForce*>(&force)) {
                if (gbsa) throw OpenMMException("B200 platform: only one GBSAOBCForce per System is supported");
                gbsa = g;
            }
            if (const NonbondedForce* nb = dynamic_cast<const NonbondedForce*>(&force)) {
                nonbonded = nb;
                if (++numNonbonded > 1) throw OpenMMException("B200 platform: only one NonbondedForce per System is supported");
                const NonbondedForce::NonbondedMethod m = nb->getNonbondedMethod();
                if (m == NonbondedForce::Ewald || m == NonbondedForce::LJPME)
                    throw OpenMMException("B200 platform: only NoCutoff, CutoffNonPeriodic, CutoffPeriodic and PME are supported");
                if (nb->getNumParticles() != system.getNumParticles()) throw OpenMMException("NonbondedForce must have exactly as many particles as the System it belongs to.");
            }
            if (force.getForceGroup() < 0 || force.getForceGroup() > 31) throw OpenMMException("B200 platform: force group out of range");
            if (dynamic_cast<const MonteCarloMembraneBarostat*>(&force)) throw OpenMMException("B200 platform: MonteCarloMembraneBarostat is not supported");
            if (const CustomTorsionForce* f = dynamic_cast<const CustomTorsionForce*>(&force)) validateCustom<CustomTorsions>(*f);
            if (const CustomBondForce* f = dynamic_cast<const CustomBondForce*>(&force)) validateCustom<CustomBonds>(*f);
            if (const CustomExternalForce* f = dynamic_cast<const CustomExternalForce*>(&force)) validateCustom<CustomExternals>(*f);
            if (const CustomAngleForce* f = dynamic_cast<const CustomAngleForce*>(&force)) validateCustom<CustomAngles>(*f);
            if (const CustomCompoundBondForce* f = dynamic_cast<const CustomCompoundBondForce*>(&force)) validateCustom<CustomCompounds>(*f);
            if (const CustomCentroidBondForce* f = dynamic_cast<const CustomCentroidBondForce*>(&force)) validateCustom<CustomCentroids>(*f);
            if (const CustomNonbondedForce* f = dynamic_cast<const CustomNonbondedForce*>(&force)) {
                validateCustomNonbonded(system, *f);
                customNonbonded.push_back(f);
            }
        }
        if (gbsa) validateGBSA(system, *gbsa, nonbonded);
        if (!customNonbonded.empty()) validateCustomNonbondedSet(customNonbonded, nonbonded, gbsa);
    }
    static void validateSystem(const System& system) {
        for (int i = 0; i < system.getNumParticles(); i++)
            if (system.isVirtualSite(i)) throw OpenMMException("B200 platform: virtual sites are not supported");
        int numCV = 0;
        vector<const Force*> forces;
        for (int f = 0; f < system.getNumForces(); f++) {
            forces.push_back(&system.getForce(f));
            if (dynamic_cast<const CustomCVForce*>(&system.getForce(f)) && ++numCV > 1)
                throw OpenMMException("B200 platform: only one CustomCVForce per System is supported");
        }
        validateForces(system, forces);
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
