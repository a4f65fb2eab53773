// plugin/tests/centroid_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the custom centroid bond tests (tests/centroid_harness.py), beside the one of the
// other custom classes (custom_capi.cpp):
//   - the plugin's own translator of a CustomCentroidBondForce expression (plugin/custom_translate.h, included, not restated);
//   - the reference's public CustomCentroidBondForce with its groups and weights, added to a System that oracle/omm_capi.cpp
//     created, and its updateParametersInContext;
//   - CustomCentroidBondForceImpl::computeNormalizedWeights of such a force.
// Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/CustomCentroidBondForce.h"
#include "openmm/TabulatedFunction.h"
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

// A CustomCentroidBondForce(ngroups, energy) with these per-bond and global parameters, no groups and no bonds; tabulated: it
// also holds a tabulated function "fn"
static CustomCentroidBondForce* centroid(int ngroups, const char* energy, const char* params, const char* globals, const double* gdefault,
                                         int periodic, int tabulated) {
    CustomCentroidBondForce* f = new CustomCentroidBondForce(ngroups, energy);
    for (const string& name : names(params)) f->addPerBondParameter(name);
    const vector<string> g = names(globals);
    for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], gdefault ? gdefault[k] : 0.0);
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    if (tabulated) f->addTabulatedFunction("fn", new Continuous1DFunction(vector<double>(4, 1.0), 0.0, 1.0));
    return f;
}

// Bonds t = 0 .. n-1 of f set (or added) to groups [n][its groups per bond], pvals [n][its number of params]
static void setBonds(CustomCentroidBondForce& f, int n, const int* groups, const double* pvals) {
    const int w = f.getNumGroupsPerBond(), np = f.getNumPerBondParameters();
    for (int t = 0; t < n; t++) {
        const vector<int> g(groups + t*w, groups + (t+1)*w);
        const vector<double> p(pvals + t*np, pvals + (t+1)*np);
        if (t < f.getNumBonds()) f.setBondParameters(t, g, p); else f.addBond(g, p);
    }
}

extern "C" {

const char* ccc_last_error() { return g_err.c_str(); }

// The programs of a centroid expression of ngroups groups per bond (the energy, then the derivatives by x1, y1, z1, x2, .. of
// the group centres), one after the other in op / arg / imm (capacity cap); counts[k] = instructions of program k.  Global
// slot s is globals[s]; tabulated: the force also holds a tabulated function "fn".  Returns the number of programs, -1 for an
// invalid expression, -2 for one the platform refuses (b200md_custom::Unsupported), -3 if cap is too small; the message is
// ccc_last_error().
int ccc_translate(int ngroups, const char* energy, const char* params, const char* globals, int tabulated, int cap, int* op, int* arg,
                  double* imm, int* counts) {
    try {
        const vector<string> g = names(globals);
        std::map<string, int> slots;
        for (size_t s = 0; s < g.size(); s++) slots[g[s]] = (int) s;
        vector<b200md_custom::Program> programs;
        std::unique_ptr<CustomCentroidBondForce> f(centroid(ngroups, energy, params, globals, nullptr, 0, tabulated));
        b200md_custom::translateCentroid(*f, slots, programs);
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

// A CustomCentroidBondForce(ngroups_per_bond, energy) with the per-bond parameters `params`, the global parameters `globals`
// (default values gdefault), ngroups groups (group g: the atoms group_atoms[group_start[g] ..] with the weights
// group_weights[group_start[g] ..], or with no weights, the masses by the Force's default, if mass[g]) and n bonds (groups
// [n][ngroups_per_bond], pvals [n][number of params]), in force group `group`.  periodic: setUsesPeriodicBoundaryConditions;
// tabulated: a tabulated function "fn"; deriv_param (may be "") asks for the energy derivative by that global.  Returns the
// index of the force in the System, or -1 with the message in ccc_last_error().
int ccc_add_force(void* system, int ngroups_per_bond, const char* energy, const char* params, const char* globals, const double* gdefault,
                  int ngroups, const int* group_start, const int* group_atoms, const double* group_weights, const int* mass,
                  int n, const int* groups, const double* pvals, int periodic, int group, int tabulated, const char* deriv_param) {
    try {
        CustomCentroidBondForce* f = centroid(ngroups_per_bond, energy, params, globals, gdefault, periodic, tabulated);
        if (deriv_param && *deriv_param) f->addEnergyParameterDerivative(deriv_param);
        for (int g = 0; g < ngroups; g++) {
            const vector<int> atoms(group_atoms + group_start[g], group_atoms + group_start[g+1]);
            f->addGroup(atoms, mass[g] ? vector<double>() : vector<double>(group_weights + group_start[g], group_weights + group_start[g+1]));
        }
        setBonds(*f, n, groups, pvals);
        f->setForceGroup(group);
        return ((System*) system)->addForce(f);
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// The CustomCentroidBondForce `index` of the System gets n bonds (groups [n][its groups per bond], pvals [n][its number of
// params]), then updateParametersInContext(context).  Returns 0, or -1 with the message in ccc_last_error().
int ccc_update_force(void* system, int index, void* context, int n, const int* groups, const double* pvals) {
    try {
        CustomCentroidBondForce& f = dynamic_cast<CustomCentroidBondForce&>(((System*) system)->getForce(index));
        setBonds(f, n, groups, pvals);
        f.updateParametersInContext(*(Context*) context);
        return 0;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

// CustomCentroidBondForceImpl::computeNormalizedWeights of the CustomCentroidBondForce `index` of the System: the weights of
// every group, one group's after the other's, into out.  Returns how many, or -1 with the message in ccc_last_error().
int ccc_normalized_weights(void* system, int index, double* out) {
    try {
        const System& s = *(System*) system;
        vector<vector<double> > weights;
        CustomCentroidBondForceImpl::computeNormalizedWeights(dynamic_cast<const CustomCentroidBondForce&>(s.getForce(index)), s, weights);
        int k = 0;
        for (const vector<double>& w : weights) for (double x : w) out[k++] = x;
        return k;
    }
    catch (const std::exception& x) { g_err = x.what(); return -1; }
}

} // extern "C"
