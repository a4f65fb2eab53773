// plugin/tests/custom_nonbonded_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the CustomNonbondedForce tests (tests/custom_nonbonded_harness.py): the reference's
// public CustomNonbondedForce with Discrete2DFunction tables, added to a System that oracle/omm_capi.cpp created, its
// updateParametersInContext, and the platform a Context of the System falls to; and, for the CPU tests of the translator,
// the plugin's programs of such a force (custom_translate.h), its energy and dE/dr evaluated by Lepton with the Reference
// platform's tabulated functions, and CustomNonbondedForceImpl::calcLongRangeCorrection.
// Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/CustomNonbondedForce.h"
#include "openmm/TabulatedFunction.h"
#include "openmm/VerletIntegrator.h"
#include "openmm/internal/CustomNonbondedForceImpl.h"
#include "../custom_translate.h"
#include <exception>
#include <set>
#include <sstream>
#include <string>
#include <vector>

using namespace OpenMM;

static std::string g_err;

static std::vector<std::string> split(const char* s) {
    std::vector<std::string> out;
    std::stringstream ss(s);
    std::string item;
    while (std::getline(ss, item, ',')) if (!item.empty()) out.push_back(item);
    return out;
}

extern "C" {

const char* cnbc_last_error() { return g_err.c_str(); }

// A CustomNonbondedForce of `energy` with the comma-separated per-particle parameters `names` (params[n][count]), method
// (CustomNonbondedForce::NonbondedMethod), cutoff, switching distance (< 0: none), long-range correction, force group, the
// excluded pairs, the comma-separated square Discrete2DFunction tables `tables` (table t: sizes[t] x sizes[t] values from
// values[start[t]]) and the comma-separated global parameters `globals` with their defaults; returns its force index or -1
int cnbc_add_force(void* sys, const char* energy, int n, const char* names, const double* params, int method, double cutoff, double sw,
                   int lrc, int group, int nexcl, const int* e1, const int* e2, const char* tables, const int* sizes, const int* start,
                   const double* values, const char* globals, const double* defaults) {
    try {
        CustomNonbondedForce* f = new CustomNonbondedForce(energy);
        const std::vector<std::string> p = split(names), t = split(tables), g = split(globals);
        for (const std::string& s : p) f->addPerParticleParameter(s);
        for (size_t k = 0; k < g.size(); k++) f->addGlobalParameter(g[k], defaults[k]);
        for (size_t k = 0; k < t.size(); k++)
            f->addTabulatedFunction(t[k], new Discrete2DFunction(sizes[k], sizes[k], std::vector<double>(values + start[k], values + start[k+1])));
        for (int i = 0; i < n; i++) f->addParticle(std::vector<double>(params + (size_t) i*p.size(), params + (size_t) (i+1)*p.size()));
        for (int k = 0; k < nexcl; k++) f->addExclusion(e1[k], e2[k]);
        f->setNonbondedMethod((CustomNonbondedForce::NonbondedMethod) method);
        f->setCutoffDistance(cutoff);
        f->setUseSwitchingFunction(sw >= 0.0);
        if (sw >= 0.0) f->setSwitchingDistance(sw);
        f->setUseLongRangeCorrection(lrc != 0);
        f->setForceGroup(group);
        return ((System*) sys)->addForce(f);
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// New per-particle parameters (params[n][count]) for force `index`, then updateParametersInContext
int cnbc_update(void* sys, int index, void* ctx, const double* params) {
    try {
        CustomNonbondedForce& f = dynamic_cast<CustomNonbondedForce&>(((System*) sys)->getForce(index));
        const int np = f.getNumPerParticleParameters();
        for (int i = 0; i < f.getNumParticles(); i++)
            f.setParticleParameters(i, std::vector<double>(params + (size_t) i*np, params + (size_t) (i+1)*np));
        f.updateParametersInContext(*(Context*) ctx);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// Interaction groups (two sets of particles) or an energy parameter derivative of global `deriv` on force `index`: the
// cases a platform may refuse
int cnbc_add_interaction_group(void* sys, int index, int n1, const int* s1, int n2, const int* s2) {
    try {
        CustomNonbondedForce& f = dynamic_cast<CustomNonbondedForce&>(((System*) sys)->getForce(index));
        f.addInteractionGroup(std::set<int>(s1, s1 + n1), std::set<int>(s2, s2 + n2));
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int cnbc_add_derivative(void* sys, int index, const char* deriv) {
    try {
        dynamic_cast<CustomNonbondedForce&>(((System*) sys)->getForce(index)).addEnergyParameterDerivative(deriv);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// A Continuous1DFunction `name` (a few values on [0, 1]) on force `index`
int cnbc_add_continuous(void* sys, int index, const char* name) {
    try {
        dynamic_cast<CustomNonbondedForce&>(((System*) sys)->getForce(index)).addTabulatedFunction(name, new Continuous1DFunction({0.0, 1.0, 0.0, 1.0}, 0.0, 1.0));
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// A Discrete1D/2D/3DFunction `name` of ndim dimensions and sizes xs, ys, zs (values x fastest) on force `index`
int cnbc_add_table(void* sys, int index, const char* name, int ndim, int xs, int ys, int zs, const double* values) {
    try {
        CustomNonbondedForce& f = dynamic_cast<CustomNonbondedForce&>(((System*) sys)->getForce(index));
        const std::vector<double> v(values, values + (size_t) xs*ys*zs);
        if (ndim == 1) f.addTabulatedFunction(name, new Discrete1DFunction(v));
        else if (ndim == 2) f.addTabulatedFunction(name, new Discrete2DFunction(xs, ys, v));
        else f.addTabulatedFunction(name, new Discrete3DFunction(xs, ys, zs, v));
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// The plugin's programs of force `index` (translateNonbonded): *nops instructions into op / arg / imm (at most cap),
// prog_start[3], and its tables (dims[4 t], start[t], values); returns 0, or -1 with the error
int cnbc_translate(void* sys, int index, int cap, int* nops, int* op, int* arg, double* imm, int* prog_start, int* ntables, int* dims,
                   int* start, double* values, int vcap) {
    try {
        const CustomNonbondedForce& f = dynamic_cast<const CustomNonbondedForce&>(((System*) sys)->getForce(index));
        std::map<std::string, int> slots;
        std::vector<b200md_custom::Program> programs;
        b200md_custom::Tables tables;
        b200md_custom::translateNonbonded(f, slots, programs, tables);
        int n = 0;
        prog_start[0] = 0;
        for (size_t q = 0; q < programs.size(); q++) {
            for (size_t k = 0; k < programs[q].op.size(); k++, n++) {
                if (n >= cap) throw OpenMMException("cnbc_translate: program buffer too small");
                op[n] = programs[q].op[k]; arg[n] = programs[q].arg[k]; imm[n] = programs[q].imm[k];
            }
            prog_start[q + 1] = n;
        }
        *nops = n;
        *ntables = tables.count();
        if ((int) tables.values.size() > vcap) throw OpenMMException("cnbc_translate: table buffer too small");
        std::copy(tables.dims.begin(), tables.dims.end(), dims);
        std::copy(tables.start.begin(), tables.start.end(), start);
        std::copy(tables.values.begin(), tables.values.end(), values);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// Lepton's value of force `index`'s energy (which = 0) or its dE/dr (which = 1) at r with the per-particle parameters p1[k]
// and p2[k] and the globals at their defaults, the tables being the Reference platform's functions
int cnbc_lepton(void* sys, int index, int which, double r, const double* p1, const double* p2, double* out) {
    try {
        const CustomNonbondedForce& f = dynamic_cast<const CustomNonbondedForce&>(((System*) sys)->getForce(index));
        std::map<std::string, Lepton::CustomFunction*> functions;
        for (int i = 0; i < f.getNumTabulatedFunctions(); i++)
            functions[f.getTabulatedFunctionName(i)] = createReferenceTabulatedFunction(f.getTabulatedFunction(i));
        Lepton::ParsedExpression e = Lepton::Parser::parse(f.getEnergyFunction(), functions).optimize();
        if (which) e = e.differentiate("r").optimize();
        std::map<std::string, double> vars;
        vars["r"] = r;
        for (int k = 0; k < f.getNumPerParticleParameters(); k++) {
            vars[f.getPerParticleParameterName(k) + "1"] = p1[k];
            vars[f.getPerParticleParameterName(k) + "2"] = p2[k];
        }
        for (int k = 0; k < f.getNumGlobalParameters(); k++) vars[f.getGlobalParameterName(k)] = f.getGlobalParameterDefaultValue(k);
        *out = e.evaluate(vars);
        for (auto& fn : functions) delete fn.second;
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// CustomNonbondedForceImpl::calcLongRangeCorrection of force `index` in the Context ctx
int cnbc_lrc(void* sys, int index, void* ctx, double* coefficient) {
    try {
        const CustomNonbondedForce& f = dynamic_cast<const CustomNonbondedForce&>(((System*) sys)->getForce(index));
        std::vector<double> derivs;
        CustomNonbondedForceImpl::calcLongRangeCorrection(f, *(Context*) ctx, *coefficient, derivs);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// The platform a Context of this System gets when none is named ("" on failure)
const char* cnbc_default_platform(void* sys) {
    static std::string name;
    try {
        VerletIntegrator integ(0.001);
        Context ctx(*(System*) sys, integ);
        name = ctx.getPlatform().getName();
    } catch (const std::exception& e) { g_err = e.what(); name = ""; }
    return name.c_str();
}

}
