// plugin/tests/custom_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the custom-force tests (tests/custom_harness.py), for every custom class
// (B200MD_CUSTOM_*; nparticles: the particles per bond of a compound bond):
//   - the plugin's own expression translator (plugin/custom_translate.h, included, not restated), so that the tests hand the
//     engine the very programs the plugin would;
//   - Lepton's ExpressionProgram::evaluate on the same expressions, with the Reference platform's own periodicdistance and
//     point functions (ReferencePointFunctions.h), the yardstick of the program interpreter;
//   - the reference's public CustomTorsionForce, CustomBondForce, CustomExternalForce, CustomAngleForce and
//     CustomCompoundBondForce, added to a System that oracle/omm_capi.cpp created, and their updateParametersInContext;
//   - the platform a Context of a System gets when none is named.
// Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/CustomTorsionForce.h"
#include "openmm/CustomBondForce.h"
#include "openmm/CustomExternalForce.h"
#include "openmm/CustomAngleForce.h"
#include "openmm/CustomCompoundBondForce.h"
#include "openmm/TabulatedFunction.h"
#include "openmm/VerletIntegrator.h"
#include "ReferencePointFunctions.h"
#include "../custom_translate.h"
#include <exception>
#include <memory>
#include <sstream>
#include <string>
#include <vector>

using namespace OpenMM;
using std::string;
using std::vector;

static string g_err;

// "a,b,c" -> {"a", "b", "c"}; "" -> {}
static vector<string> names(const char* list) {
    vector<string> out;
    std::stringstream ss(list ? list : "");
    string item;
    while (std::getline(ss, item, ',')) if (!item.empty()) out.push_back(item);
    return out;
}

// the variables of a class but compound bonds, the name of its Force and of its terms in messages
static vector<string> variables(int cls) {
    if (cls == B200MD_CUSTOM_BOND) return {"r"};
    if (cls == B200MD_CUSTOM_EXTERNAL) return {"x", "y", "z"};
    return {"theta"};
}
static const char* const FORCE_NAME[] = {"CustomTorsionForce", "CustomBondForce", "CustomExternalForce", "CustomAngleForce"};
static const char* const PER_TERM[] = {"torsion", "bond", "particle", "angle"};

// A CustomCompoundBondForce(nparticles, energy) with these per-bond and global parameters and no bonds; tabulated: it also
// holds a tabulated function "fn"
static CustomCompoundBondForce* compound(int nparticles, const char* energy, const char* params, const char* globals, const double* gdefault,
                                         int periodic, int tabulated) {
    CustomCompoundBondForce* f = new CustomCompoundBondForce(nparticles, energy);
    for (const string& name : names(params)) f->addPerBondParameter(name);
    const vector<string> g = names(globals);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault ? gdefault[k] : 0.0);
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    if (tabulated) f->addTabulatedFunction("fn", new Continuous1DFunction(vector<double>(4, 1.0), 0.0, 1.0));
    return f;
}

// What the five Force classes name differently: a term's atoms a[0 .. width-1], its per-term parameters, the term count
static void addParam(CustomTorsionForce& f, const string& n) { f.addPerTorsionParameter(n); }
static void addParam(CustomBondForce& f, const string& n) { f.addPerBondParameter(n); }
static void addParam(CustomExternalForce& f, const string& n) { f.addPerParticleParameter(n); }
static void addParam(CustomAngleForce& f, const string& n) { f.addPerAngleParameter(n); }
static void setTerm(CustomTorsionForce& f, int t, const int* a, int, const vector<double>& p) {
    if (t < f.getNumTorsions()) f.setTorsionParameters(t, a[0], a[1], a[2], a[3], p); else f.addTorsion(a[0], a[1], a[2], a[3], p);
}
static void setTerm(CustomBondForce& f, int t, const int* a, int, const vector<double>& p) {
    if (t < f.getNumBonds()) f.setBondParameters(t, a[0], a[1], p); else f.addBond(a[0], a[1], p);
}
static void setTerm(CustomExternalForce& f, int t, const int* a, int, const vector<double>& p) {
    if (t < f.getNumParticles()) f.setParticleParameters(t, a[0], p); else f.addParticle(a[0], p);
}
static void setTerm(CustomAngleForce& f, int t, const int* a, int, const vector<double>& p) {
    if (t < f.getNumAngles()) f.setAngleParameters(t, a[0], a[1], a[2], p); else f.addAngle(a[0], a[1], a[2], p);
}
static void setTerm(CustomCompoundBondForce& f, int t, const int* a, int w, const vector<double>& p) {
    const vector<int> atoms(a, a + w);
    if (t < f.getNumBonds()) f.setBondParameters(t, atoms, p); else f.addBond(atoms, p);
}
static int numParams(const CustomTorsionForce& f) { return f.getNumPerTorsionParameters(); }
static int numParams(const CustomBondForce& f) { return f.getNumPerBondParameters(); }
static int numParams(const CustomExternalForce& f) { return f.getNumPerParticleParameters(); }
static int numParams(const CustomAngleForce& f) { return f.getNumPerAngleParameters(); }
static int numParams(const CustomCompoundBondForce& f) { return f.getNumPerBondParameters(); }

// Terms t = 0 .. n-1 of f set (or added) to atoms [n][w], pvals [n][its number of params]
template<class F> void setTerms(F& f, int n, int w, const int* atoms, const double* pvals) {
    const int np = numParams(f);
    for (int t = 0; t < n; t++) setTerm(f, t, atoms + t*w, w, vector<double>(pvals + t*np, pvals + (t+1)*np));
}

// f (one of the four classes but compound bonds) with its parameters, globals, periodic flag and energy derivative
template<class F> F* withParameters(F* f, const char* params, const char* globals, const double* gdefault, int periodic, const char* deriv_param) {
    for (const string& name : names(params)) addParam(*f, name);
    const vector<string> g = names(globals);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault[k]);
    if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    return f;
}

// the terms of class cls per term
static int width(int cls, int nparticles) {
    const int w[] = {4, 2, 1, 3};
    return cls == B200MD_CUSTOM_COMPOUND ? nparticles : w[cls];
}

extern "C" {

const char* cc_last_error() { return g_err.c_str(); }

// The programs of `energy` for class cls (the energy, then one derivative per variable: a compound bond's by x1, y1, z1, x2,
// ..), one after the other in op / arg / imm (capacity cap); counts[k] = instructions of program k.  Global slot s is
// globals[s]; tabulated: a compound force also holds a tabulated function "fn".  Returns the number of programs, -1 for an
// invalid expression (e.g. an unknown variable), -2 for one the platform refuses (b200md_custom::Unsupported), -3 if cap is
// too small; the message is cc_last_error().
int cc_translate(int cls, int nparticles, const char* energy, const char* params, const char* globals, int tabulated, int cap, int* op, int* arg,
                 double* imm, int* counts) {
    try {
        const vector<string> g = names(globals);
        std::map<string, int> slots;
        for (size_t s = 0; s < g.size(); s++) slots[g[s]] = (int) s;
        vector<b200md_custom::Program> programs;
        if (cls == B200MD_CUSTOM_COMPOUND) {
            std::unique_ptr<CustomCompoundBondForce> f(compound(nparticles, energy, params, globals, nullptr, 0, tabulated));
            b200md_custom::translateCompound(*f, slots, programs);
        }
        else
            b200md_custom::translateExpression(energy, variables(cls), FORCE_NAME[cls], PER_TERM[cls], cls == B200MD_CUSTOM_EXTERNAL, names(params),
                                               g, slots, programs);
        int k = 0;
        for (size_t q = 0; q < programs.size(); q++) {
            const b200md_custom::Program& p = programs[q];
            if (k + (int) p.op.size() > cap) { g_err = "capacity"; return -3; }
            for (size_t i = 0; i < p.op.size(); i++, k++) { op[k] = p.op[i]; arg[k] = p.arg[i]; imm[k] = p.imm[i]; }
            counts[q] = (int) p.op.size();
        }
        return (int) programs.size();
    }
    catch (const b200md_custom::Unsupported& x) { g_err = x.what(); return -2; }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// Lepton's own value of the energy (which = 0) or of its derivative by variable which-1 of `energy` (class cls), parsed,
// optimised and differentiated as custom_translate.h does, through ExpressionProgram::evaluate at the variables vars.  An
// external's periodicdistance and a compound bond's point functions (prepared by prepareExpression; periodic or not) are the
// Reference platform's, in the box whose vectors are box[0..2], box[3..5], box[6..8].
int cc_lepton_eval(int cls, int nparticles, const char* energy, int which, const double* vars, const double* box, int periodic, const char* params,
                   const double* pvals, const char* globals, const double* gvals, double* out) {
    try {
        Vec3 boxVectors[3] = {Vec3(box[0], box[1], box[2]), Vec3(box[3], box[4], box[5]), Vec3(box[6], box[7], box[8])};
        Vec3* handle = boxVectors;
        ReferencePointDistanceFunction periodicDistance(true, &handle), distance(periodic != 0, &handle);
        ReferencePointAngleFunction angle(periodic != 0, &handle);
        ReferencePointDihedralFunction dihedral(periodic != 0, &handle);
        std::map<string, Lepton::CustomFunction*> functions;
        vector<string> v;
        Lepton::ParsedExpression expr;
        if (cls == B200MD_CUSTOM_COMPOUND) {
            functions["pointdistance"] = &distance; functions["pointangle"] = &angle; functions["pointdihedral"] = &dihedral;
            std::unique_ptr<CustomCompoundBondForce> f(compound(nparticles, energy, params, globals, nullptr, periodic, 0));
            expr = CustomCompoundBondForceImpl::prepareExpression(*f, functions);
            for (int i = 1; i <= nparticles; i++)
                for (const char* axis : {"x", "y", "z"}) v.push_back(axis + std::to_string(i));
        }
        else {
            if (cls == B200MD_CUSTOM_EXTERNAL) functions["periodicdistance"] = &periodicDistance;
            expr = Lepton::Parser::parse(energy, functions).optimize();
            v = variables(cls);
        }
        if (which > 0) expr = expr.differentiate(v[which-1]).optimize();
        std::map<string, double> values;
        for (size_t k = 0; k < v.size(); k++) values[v[k]] = vars[k];
        const vector<string> p = names(params), g = names(globals);
        for (size_t k = 0; k < g.size(); k++) values[g[k]] = gvals[k];
        for (size_t k = 0; k < p.size(); k++) values[p[k]] = pvals[k];
        *out = expr.createProgram().evaluate(values);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// A Force of class cls (energy) with the per-term parameters `params`, the global parameters `globals` (default values
// gdefault) and n terms (atoms [n][the class's atoms per term], pvals [n][number of params]), in force group `group`.
// periodic: setUsesPeriodicBoundaryConditions (not for externals); deriv_param (may be "") asks for the energy derivative by
// that global (not for externals); tabulated: a compound force also holds a tabulated function "fn".  Returns the index of the
// force in the System.
int cc_add_force(void* system, int cls, int nparticles, const char* energy, const char* params, const char* globals, const double* gdefault,
                 int n, const int* atoms, const double* pvals, int periodic, int group, int tabulated, const char* deriv_param) {
    Force* force;
    const int w = width(cls, nparticles);
    if (cls == B200MD_CUSTOM_TORSION) {
        CustomTorsionForce* f = withParameters(new CustomTorsionForce(energy), params, globals, gdefault, periodic, deriv_param);
        setTerms(*f, n, w, atoms, pvals); force = f;
    }
    else if (cls == B200MD_CUSTOM_BOND) {
        CustomBondForce* f = withParameters(new CustomBondForce(energy), params, globals, gdefault, periodic, deriv_param);
        setTerms(*f, n, w, atoms, pvals); force = f;
    }
    else if (cls == B200MD_CUSTOM_EXTERNAL) {
        CustomExternalForce* f = new CustomExternalForce(energy);
        for (const string& name : names(params)) f->addPerParticleParameter(name);
        const vector<string> g = names(globals);
        for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault[k]);
        setTerms(*f, n, w, atoms, pvals); force = f;
    }
    else if (cls == B200MD_CUSTOM_ANGLE) {
        CustomAngleForce* f = withParameters(new CustomAngleForce(energy), params, globals, gdefault, periodic, deriv_param);
        setTerms(*f, n, w, atoms, pvals); force = f;
    }
    else {
        CustomCompoundBondForce* f = compound(nparticles, energy, params, globals, gdefault, periodic, tabulated);
        if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
        setTerms(*f, n, w, atoms, pvals); force = f;
    }
    force->setForceGroup(group);
    return ((System*) system)->addForce(force);
}

// Force `index` of the System (of class cls) gets n terms atoms [n][its atoms per term], pvals [n][its number of params], then
// updateParametersInContext(context).  Returns 0, or -1 with the message in cc_last_error().
int cc_update_force(void* system, int cls, int index, void* context, int n, const int* atoms, const double* pvals) {
    try {
        Force& force = ((System*) system)->getForce(index);
        Context& c = *(Context*) context;
        if (cls == B200MD_CUSTOM_TORSION) { CustomTorsionForce& f = dynamic_cast<CustomTorsionForce&>(force); setTerms(f, n, 4, atoms, pvals); f.updateParametersInContext(c); }
        else if (cls == B200MD_CUSTOM_BOND) { CustomBondForce& f = dynamic_cast<CustomBondForce&>(force); setTerms(f, n, 2, atoms, pvals); f.updateParametersInContext(c); }
        else if (cls == B200MD_CUSTOM_EXTERNAL) { CustomExternalForce& f = dynamic_cast<CustomExternalForce&>(force); setTerms(f, n, 1, atoms, pvals); f.updateParametersInContext(c); }
        else if (cls == B200MD_CUSTOM_ANGLE) { CustomAngleForce& f = dynamic_cast<CustomAngleForce&>(force); setTerms(f, n, 3, atoms, pvals); f.updateParametersInContext(c); }
        else {
            CustomCompoundBondForce& f = dynamic_cast<CustomCompoundBondForce&>(force);
            setTerms(f, n, f.getNumParticlesPerBond(), atoms, pvals);
            f.updateParametersInContext(c);
        }
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// The platform a Context of this System gets when none is named (the fastest one whose contextCreated accepts it), or "" with
// the message in cc_last_error().
const char* cc_default_platform(void* system) {
    static string name;
    try {
        VerletIntegrator integrator(0.001);
        Context context(*(System*) system, integrator);
        name = context.getPlatform().getName();
    }
    catch (const std::exception& x) { g_err = x.what(); name = ""; }
    return name.c_str();
}

} // extern "C"
