// plugin/tests/custom_torsion_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the custom-torsion tests (tests/custom_torsion_harness.py):
//   - the plugin's own expression translator (plugin/custom_translate.h, included, not restated), so that the tests hand the
//     engine the very programs the plugin would;
//   - Lepton's ExpressionProgram::evaluate on the same expressions, the yardstick of the program interpreter;
//   - the reference's public CustomTorsionForce, added to a System that oracle/omm_capi.cpp created, and its
//     updateParametersInContext.
// Built by plugin/Makefile (target `reftests`) against the staged headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/CustomTorsionForce.h"
#include "openmm/VerletIntegrator.h"
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

extern "C" {

const char* ct_last_error() { return g_err.c_str(); }

// The energy program and the dE/dtheta program of `energy`, one after the other in op / arg / imm (capacity cap); global
// slot s is globals[s].  Returns 0, -1 for an invalid expression (e.g. an unknown variable), -2 for one the platform refuses
// (b200md_custom::Unsupported), -3 if cap is too small; the message is ct_last_error().
int ct_translate(const char* energy, const char* params, const char* globals, int cap, int* op, int* arg, double* imm, int* nEnergy, int* nDeriv) {
    try {
        const std::vector<std::string> g = names(globals);
        std::map<std::string, int> slots;
        for (size_t s = 0; s < g.size(); s++) slots[g[s]] = (int) s;
        b200md_custom::Program e, d;
        b200md_custom::translateExpression(energy, names(params), g, slots, e, d);
        if ((int) (e.op.size() + d.op.size()) > cap) { g_err = "capacity"; return -3; }
        int k = 0;
        for (const b200md_custom::Program* p : {&e, &d})
            for (size_t i = 0; i < p->op.size(); i++, k++) { op[k] = p->op[i]; arg[k] = p->arg[i]; imm[k] = p->imm[i]; }
        *nEnergy = (int) e.op.size(); *nDeriv = (int) d.op.size();
        return 0;
    }
    catch (const b200md_custom::Unsupported& x) { g_err = x.what(); return -2; }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// Lepton's own value of the energy (deriv = 0) or of dE/dtheta (deriv = 1) of `energy`, parsed, optimised and differentiated
// as custom_translate.h does, through ExpressionProgram::evaluate.
int ct_lepton_eval(const char* energy, int deriv, double theta, const char* params, const double* pvals, const char* globals, const double* gvals, double* out) {
    try {
        Lepton::ParsedExpression expr = Lepton::Parser::parse(energy).optimize();
        if (deriv) expr = expr.differentiate("theta").optimize();
        std::map<std::string, double> vars;
        vars["theta"] = theta;
        const std::vector<std::string> p = names(params), g = names(globals);
        for (size_t k = 0; k < g.size(); k++) vars[g[k]] = gvals[k];
        for (size_t k = 0; k < p.size(); k++) vars[p[k]] = pvals[k];
        *out = expr.createProgram().evaluate(vars);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// A CustomTorsionForce(energy) with the per-torsion parameters `params`, the global parameters `globals` (default values
// gdefault) and n torsions (atoms [n][4], pvals [n][number of params]); deriv_param (may be "") asks for the energy
// derivative by that global.  Returns the index of the force in the System.
int ct_add_custom_torsions(void* system, const char* energy, const char* params, const char* globals, const double* gdefault,
                           int n, const int* atoms, const double* pvals, int periodic, int group, const char* deriv_param) {
    CustomTorsionForce* f = new CustomTorsionForce(energy);
    const std::vector<std::string> p = names(params), g = names(globals);
    for (const std::string& name : p) f->addPerTorsionParameter(name);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault[k]);
    if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
    for (int t = 0; t < n; t++)
        f->addTorsion(atoms[4*t], atoms[4*t+1], atoms[4*t+2], atoms[4*t+3], std::vector<double>(pvals + t*p.size(), pvals + (t+1)*p.size()));
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// Force `index` of the System (a CustomTorsionForce) gets n torsions atoms [n][4], pvals [n][its number of params], then
// updateParametersInContext(context).  Returns 0, or -1 with the message in ct_last_error().
int ct_update_custom_torsions(void* system, int index, void* context, int n, const int* atoms, const double* pvals) {
    try {
        CustomTorsionForce& f = dynamic_cast<CustomTorsionForce&>(((System*) system)->getForce(index));
        const int np = f.getNumPerTorsionParameters();
        for (int t = 0; t < n; t++) {
            const std::vector<double> v(pvals + t*np, pvals + (t+1)*np);
            if (t < f.getNumTorsions()) f.setTorsionParameters(t, atoms[4*t], atoms[4*t+1], atoms[4*t+2], atoms[4*t+3], v);
            else f.addTorsion(atoms[4*t], atoms[4*t+1], atoms[4*t+2], atoms[4*t+3], v);
        }
        f.updateParametersInContext(*(Context*) context);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// The platform a Context of this System gets when none is named (the fastest one whose contextCreated accepts it), or "" with
// the message in ct_last_error().
const char* ct_default_platform(void* system) {
    static std::string name;
    try {
        VerletIntegrator integrator(0.001);
        Context context(*(System*) system, integrator);
        name = context.getPlatform().getName();
    }
    catch (const std::exception& x) { g_err = x.what(); name = ""; }
    return name.c_str();
}

} // extern "C"
