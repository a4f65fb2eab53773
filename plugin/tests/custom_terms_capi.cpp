// plugin/tests/custom_terms_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the custom-bond and custom-external tests (tests/custom_terms_harness.py):
//   - the plugin's own expression translator (plugin/custom_translate.h, included, not restated) for the three classes, so
//     that the tests hand the engine the very programs the plugin would;
//   - Lepton's ExpressionProgram::evaluate on the same expressions, with the Reference platform's own periodicdistance
//     (ReferencePointDistanceFunction), the yardstick of the program interpreter;
//   - the reference's public CustomBondForce and CustomExternalForce, added to a System that oracle/omm_capi.cpp created, and
//     their updateParametersInContext.
// Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/CustomBondForce.h"
#include "openmm/CustomExternalForce.h"
#include "ReferencePointFunctions.h"
#include "../custom_translate.h"
#include <cstring>
#include <exception>
#include <sstream>
#include <string>
#include <vector>

using namespace OpenMM;

static std::string g_err;

// "a,b,c" -> {"a", "b", "c"}; "" -> {}
static std::vector<std::string> names(const char* list) {
    std::vector<std::string> out;
    std::stringstream ss(list ? list : "");
    std::string item;
    while (std::getline(ss, item, ',')) if (!item.empty()) out.push_back(item);
    return out;
}

// the variables of a class (B200MD_CUSTOM_*)
static std::vector<std::string> variables(int cls) {
    if (cls == B200MD_CUSTOM_TORSION) return {"theta"};
    if (cls == B200MD_CUSTOM_BOND) return {"r"};
    return {"x", "y", "z"};
}
static const char* forceName(int cls) {
    return cls == B200MD_CUSTOM_TORSION ? "CustomTorsionForce" : cls == B200MD_CUSTOM_BOND ? "CustomBondForce" : "CustomExternalForce";
}

extern "C" {

const char* cterm_last_error() { return g_err.c_str(); }

// The programs of `energy` for class cls (the energy, then one derivative per variable), one after the other in op / arg /
// imm (capacity cap); counts[k] = instructions of program k.  Global slot s is globals[s].  Returns the number of programs,
// -1 for an invalid expression (e.g. an unknown variable), -2 for one the platform refuses (b200md_custom::Unsupported), -3 if
// cap is too small; the message is cterm_last_error().
int cterm_translate(int cls, const char* energy, const char* params, const char* globals, int cap, int* op, int* arg, double* imm, int* counts) {
    try {
        const std::vector<std::string> g = names(globals);
        std::map<std::string, int> slots;
        for (size_t s = 0; s < g.size(); s++) slots[g[s]] = (int) s;
        std::vector<b200md_custom::Program> programs;
        b200md_custom::translateExpression(energy, variables(cls), forceName(cls), "term", cls == B200MD_CUSTOM_EXTERNAL, names(params), g,
                                           slots, programs);
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
// optimised and differentiated as custom_translate.h does, through ExpressionProgram::evaluate at the variables vars; an
// external's periodicdistance is the Reference platform's, in the box whose vectors are box[0..2], box[3..5], box[6..8].
int cterm_lepton_eval(int cls, const char* energy, int which, const double* vars, const double* box, const char* params, const double* pvals,
                      const char* globals, const double* gvals, double* out) {
    try {
        Vec3 boxVectors[3] = {Vec3(box[0], box[1], box[2]), Vec3(box[3], box[4], box[5]), Vec3(box[6], box[7], box[8])};
        Vec3* handle = boxVectors;
        ReferencePointDistanceFunction periodicDistance(true, &handle);
        std::map<std::string, Lepton::CustomFunction*> functions;
        if (cls == B200MD_CUSTOM_EXTERNAL) functions["periodicdistance"] = &periodicDistance;
        Lepton::ParsedExpression expr = Lepton::Parser::parse(energy, functions).optimize();
        const std::vector<std::string> v = variables(cls);
        if (which > 0) expr = expr.differentiate(v[which-1]).optimize();
        std::map<std::string, double> values;
        for (size_t k = 0; k < v.size(); k++) values[v[k]] = vars[k];
        const std::vector<std::string> p = names(params), g = names(globals);
        for (size_t k = 0; k < g.size(); k++) values[g[k]] = gvals[k];
        for (size_t k = 0; k < p.size(); k++) values[p[k]] = pvals[k];
        *out = expr.createProgram().evaluate(values);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// A CustomBondForce(energy) with the per-bond parameters `params`, the global parameters `globals` (default values
// gdefault) and n bonds (atoms [n][2], pvals [n][number of params]); deriv_param (may be "") asks for the energy derivative
// by that global.  Returns the index of the force in the System.
int cterm_add_custom_bonds(void* system, const char* energy, const char* params, const char* globals, const double* gdefault,
                           int n, const int* atoms, const double* pvals, int periodic, int group, const char* deriv_param) {
    CustomBondForce* f = new CustomBondForce(energy);
    const std::vector<std::string> p = names(params), g = names(globals);
    for (const std::string& name : p) f->addPerBondParameter(name);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault[k]);
    if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
    for (int t = 0; t < n; t++) f->addBond(atoms[2*t], atoms[2*t+1], std::vector<double>(pvals + t*p.size(), pvals + (t+1)*p.size()));
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// A CustomExternalForce(energy) on n particles (atoms [n], pvals [n][number of params]).  Returns its index in the System.
int cterm_add_custom_externals(void* system, const char* energy, const char* params, const char* globals, const double* gdefault,
                               int n, const int* atoms, const double* pvals, int group) {
    CustomExternalForce* f = new CustomExternalForce(energy);
    const std::vector<std::string> p = names(params), g = names(globals);
    for (const std::string& name : p) f->addPerParticleParameter(name);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault[k]);
    for (int t = 0; t < n; t++) f->addParticle(atoms[t], std::vector<double>(pvals + t*p.size(), pvals + (t+1)*p.size()));
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// Force `index` of the System (a CustomBondForce) gets n bonds atoms [n][2], pvals [n][its number of params], then
// updateParametersInContext(context).  Returns 0, or -1 with the message in cterm_last_error().
int cterm_update_custom_bonds(void* system, int index, void* context, int n, const int* atoms, const double* pvals) {
    try {
        CustomBondForce& f = dynamic_cast<CustomBondForce&>(((System*) system)->getForce(index));
        const int np = f.getNumPerBondParameters();
        for (int t = 0; t < n; t++) {
            const std::vector<double> v(pvals + t*np, pvals + (t+1)*np);
            if (t < f.getNumBonds()) f.setBondParameters(t, atoms[2*t], atoms[2*t+1], v);
            else f.addBond(atoms[2*t], atoms[2*t+1], v);
        }
        f.updateParametersInContext(*(Context*) context);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// The same for a CustomExternalForce: n particles atoms [n], pvals [n][its number of params].
int cterm_update_custom_externals(void* system, int index, void* context, int n, const int* atoms, const double* pvals) {
    try {
        CustomExternalForce& f = dynamic_cast<CustomExternalForce&>(((System*) system)->getForce(index));
        const int np = f.getNumPerParticleParameters();
        for (int t = 0; t < n; t++) {
            const std::vector<double> v(pvals + t*np, pvals + (t+1)*np);
            if (t < f.getNumParticles()) f.setParticleParameters(t, atoms[t], v);
            else f.addParticle(atoms[t], v);
        }
        f.updateParametersInContext(*(Context*) context);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

} // extern "C"
