// plugin/tests/custom_compound_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the custom-angle and custom-compound-bond tests (tests/custom_compound_harness.py):
//   - the plugin's own expression translator (plugin/custom_translate.h, included, not restated) for the two classes;
//   - Lepton's ExpressionProgram::evaluate on the same expressions, a compound bond's prepared by
//     CustomCompoundBondForceImpl::prepareExpression with the Reference platform's own point functions
//     (ReferencePointFunctions.h), the yardstick of the program interpreter;
//   - the reference's public CustomAngleForce and CustomCompoundBondForce, added to a System that oracle/omm_capi.cpp
//     created, and their updateParametersInContext.
// Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/CustomAngleForce.h"
#include "openmm/CustomCompoundBondForce.h"
#include "openmm/TabulatedFunction.h"
#include "ReferencePointFunctions.h"
#include "../custom_translate.h"
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

// A CustomCompoundBondForce(nparticles, energy) with these per-bond and global parameters and no bonds
static CustomCompoundBondForce* compound(int nparticles, const char* energy, const char* params, const char* globals, const double* gdefault,
                                         int periodic) {
    CustomCompoundBondForce* f = new CustomCompoundBondForce(nparticles, energy);
    for (const std::string& name : names(params)) f->addPerBondParameter(name);
    const std::vector<std::string> g = names(globals);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault ? gdefault[k] : 0.0);
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    return f;
}

static int flatten(const std::vector<b200md_custom::Program>& programs, int cap, int* op, int* arg, double* imm, int* counts) {
    int k = 0;
    for (size_t q = 0; q < programs.size(); q++) {
        const b200md_custom::Program& p = programs[q];
        if (k + (int) p.op.size() > cap) { g_err = "capacity"; return -3; }
        for (size_t i = 0; i < p.op.size(); i++, k++) { op[k] = p.op[i]; arg[k] = p.arg[i]; imm[k] = p.imm[i]; }
        counts[q] = (int) p.op.size();
    }
    return (int) programs.size();
}

extern "C" {

const char* ccomp_last_error() { return g_err.c_str(); }

// The programs of a CustomAngleForce `energy` (the energy, dE/dtheta) or, with nparticles > 0, of a CustomCompoundBondForce
// (the energy, then the derivatives by x1, y1, z1, x2, ..), one after the other in op / arg / imm (capacity cap); counts[k] =
// instructions of program k.  Global slot s is globals[s].  tabulated: the compound force also holds a tabulated function
// "fn".  Returns the number of programs, -1 for an invalid expression, -2 for one the platform refuses
// (b200md_custom::Unsupported), -3 if cap is too small; the message is ccomp_last_error().
int ccomp_translate(int nparticles, const char* energy, const char* params, const char* globals, int tabulated, int cap, int* op, int* arg,
                    double* imm, int* counts) {
    try {
        const std::vector<std::string> g = names(globals);
        std::map<std::string, int> slots;
        for (size_t s = 0; s < g.size(); s++) slots[g[s]] = (int) s;
        std::vector<b200md_custom::Program> programs;
        if (nparticles <= 0)
            b200md_custom::translateExpression(energy, std::vector<std::string>(1, "theta"), "CustomAngleForce", "angle", false, names(params), g,
                                               slots, programs);
        else {
            CustomCompoundBondForce* f = compound(nparticles, energy, params, globals, nullptr, 0);
            if (tabulated) f->addTabulatedFunction("fn", new Continuous1DFunction(std::vector<double>(4, 1.0), 0.0, 1.0));
            try { b200md_custom::translateCompound(*f, slots, programs); }
            catch (...) { delete f; throw; }
            delete f;
        }
        return flatten(programs, cap, op, arg, imm, counts);
    }
    catch (const b200md_custom::Unsupported& x) { g_err = x.what(); return -2; }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// Lepton's own value of the energy (which = 0) or of its derivative by variable which-1, parsed, optimised and differentiated
// as custom_translate.h does, through ExpressionProgram::evaluate at the variables vars.  nparticles <= 0: a CustomAngleForce
// expression of theta.  Otherwise a compound bond's, prepared by prepareExpression with the Reference platform's point
// functions, periodic or not, in the box whose vectors are box[0..2], box[3..5], box[6..8].
int ccomp_lepton_eval(int nparticles, const char* energy, int which, const double* vars, const double* box, int periodic, const char* params,
                      const double* pvals, const char* globals, const double* gvals, double* out) {
    try {
        Vec3 boxVectors[3] = {Vec3(box[0], box[1], box[2]), Vec3(box[3], box[4], box[5]), Vec3(box[6], box[7], box[8])};
        Vec3* handle = boxVectors;
        ReferencePointDistanceFunction distance(periodic != 0, &handle);
        ReferencePointAngleFunction angle(periodic != 0, &handle);
        ReferencePointDihedralFunction dihedral(periodic != 0, &handle);
        std::vector<std::string> v;
        Lepton::ParsedExpression expr;
        if (nparticles <= 0) {
            v.push_back("theta");
            expr = Lepton::Parser::parse(energy).optimize();
        }
        else {
            std::map<std::string, Lepton::CustomFunction*> functions;
            functions["pointdistance"] = &distance; functions["pointangle"] = &angle; functions["pointdihedral"] = &dihedral;
            CustomCompoundBondForce* f = compound(nparticles, energy, params, globals, nullptr, periodic);
            try { expr = CustomCompoundBondForceImpl::prepareExpression(*f, functions); }
            catch (...) { delete f; throw; }
            delete f;
            for (int i = 1; i <= nparticles; i++)
                for (const char* axis : {"x", "y", "z"}) v.push_back(axis + std::to_string(i));
        }
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

// A CustomAngleForce(energy) with the per-angle parameters `params`, the global parameters `globals` (default values
// gdefault) and n angles (atoms [n][3], pvals [n][number of params]); deriv_param (may be "") asks for the energy derivative
// by that global.  Returns the index of the force in the System.
int ccomp_add_custom_angles(void* system, const char* energy, const char* params, const char* globals, const double* gdefault,
                            int n, const int* atoms, const double* pvals, int periodic, int group, const char* deriv_param) {
    CustomAngleForce* f = new CustomAngleForce(energy);
    const std::vector<std::string> p = names(params), g = names(globals);
    for (const std::string& name : p) f->addPerAngleParameter(name);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault[k]);
    if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
    for (int t = 0; t < n; t++)
        f->addAngle(atoms[3*t], atoms[3*t+1], atoms[3*t+2], std::vector<double>(pvals + t*p.size(), pvals + (t+1)*p.size()));
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// A CustomCompoundBondForce(nparticles, energy) with n bonds (atoms [n][nparticles], pvals [n][number of params]); tabulated:
// it also holds a tabulated function "fn".  Returns its index in the System.
int ccomp_add_compound(void* system, int nparticles, const char* energy, const char* params, const char* globals, const double* gdefault,
                       int n, const int* atoms, const double* pvals, int periodic, int group, int tabulated, const char* deriv_param) {
    CustomCompoundBondForce* f = compound(nparticles, energy, params, globals, gdefault, periodic);
    const size_t np = names(params).size();
    if (tabulated) f->addTabulatedFunction("fn", new Continuous1DFunction(std::vector<double>(4, 1.0), 0.0, 1.0));
    if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
    for (int t = 0; t < n; t++)
        f->addBond(std::vector<int>(atoms + t*nparticles, atoms + (t+1)*nparticles), std::vector<double>(pvals + t*np, pvals + (t+1)*np));
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// Force `index` of the System (a CustomAngleForce) gets n angles atoms [n][3], pvals [n][its number of params], then
// updateParametersInContext(context).  Returns 0, or -1 with the message in ccomp_last_error().
int ccomp_update_custom_angles(void* system, int index, void* context, int n, const int* atoms, const double* pvals) {
    try {
        CustomAngleForce& f = dynamic_cast<CustomAngleForce&>(((System*) system)->getForce(index));
        const int np = f.getNumPerAngleParameters();
        for (int t = 0; t < n; t++) {
            const std::vector<double> v(pvals + t*np, pvals + (t+1)*np);
            if (t < f.getNumAngles()) f.setAngleParameters(t, atoms[3*t], atoms[3*t+1], atoms[3*t+2], v);
            else f.addAngle(atoms[3*t], atoms[3*t+1], atoms[3*t+2], v);
        }
        f.updateParametersInContext(*(Context*) context);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// The same for a CustomCompoundBondForce: n bonds atoms [n][its particles per bond].
int ccomp_update_compound(void* system, int index, void* context, int n, const int* atoms, const double* pvals) {
    try {
        CustomCompoundBondForce& f = dynamic_cast<CustomCompoundBondForce&>(((System*) system)->getForce(index));
        const int np = f.getNumPerBondParameters(), w = f.getNumParticlesPerBond();
        for (int t = 0; t < n; t++) {
            const std::vector<double> v(pvals + t*np, pvals + (t+1)*np);
            const std::vector<int> a(atoms + t*w, atoms + (t+1)*w);
            if (t < f.getNumBonds()) f.setBondParameters(t, a, v);
            else f.addBond(a, v);
        }
        f.updateParametersInContext(*(Context*) context);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

} // extern "C"
