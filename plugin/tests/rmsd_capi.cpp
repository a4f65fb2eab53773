// plugin/tests/rmsd_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the RMSDForce and CustomCVForce tests (tests/rmsd_harness.py): the reference's public
// RMSDForce, added to a System that oracle/omm_capi.cpp created, its updateParametersInContext, and a stand-alone evaluation of
// one RMSDForce on a named platform; a CustomCVForce with RMSD, centroid-distance, torsion and CustomNonbondedForce variables,
// a Continuous2DFunction, its collective variable values and updateParametersInContext.  Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/Platform.h"
#include "openmm/State.h"
#include "openmm/RMSDForce.h"
#include "openmm/CustomCVForce.h"
#include "openmm/CustomCentroidBondForce.h"
#include "openmm/CustomTorsionForce.h"
#include "openmm/CustomNonbondedForce.h"
#include "openmm/TabulatedFunction.h"
#include "openmm/VerletIntegrator.h"
#include <exception>
#include <map>
#include <string>
#include <vector>

using namespace OpenMM;

static std::string g_err;

static std::vector<Vec3> vec3(int n, const double* x) {
    std::vector<Vec3> v(n);
    for (int i = 0; i < n; i++) v[i] = Vec3(x[3*i], x[3*i+1], x[3*i+2]);
    return v;
}

extern "C" {

const char* rmc_last_error() { return g_err.c_str(); }

// An RMSDForce over the n particles (n = 0: every particle) with the nref reference positions ref[3 nref], in force group
// `group`, added to the System; returns its force index or -1
int rmc_add_force(void* sys, int n, const int* particles, int nref, const double* ref, int group) {
    try {
        RMSDForce* f = new RMSDForce(vec3(nref, ref), std::vector<int>(particles, particles + n));
        f->setForceGroup(group);
        return ((System*) sys)->addForce(f);
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// New particles and reference positions for force `index`, then updateParametersInContext
int rmc_update(void* sys, int index, void* ctx, int n, const int* particles, int nref, const double* ref) {
    try {
        RMSDForce& f = dynamic_cast<RMSDForce&>(((System*) sys)->getForce(index));
        f.setParticles(std::vector<int>(particles, particles + n));
        f.setReferencePositions(vec3(nref, ref));
        f.updateParametersInContext(*(Context*) ctx);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// The platform a Context of this System gets when none is named ("" on failure)
const char* rmc_default_platform(void* sys) {
    static std::string name;
    try {
        VerletIntegrator integ(0.001);
        Context ctx(*(System*) sys, integ);
        name = ctx.getPlatform().getName();
    } catch (const std::exception& e) { g_err = e.what(); name = ""; }
    return name.c_str();
}

// One RMSDForce alone in a System of natoms unit masses, on `platform` (property Precision = precision unless empty), at the
// positions pos[3 natoms]: its energy and forces[3 natoms]
int rmc_evaluate(int natoms, const double* pos, const double* ref, int n, const int* particles, const char* platform,
                 const char* precision, double* energy, double* forces) {
    try {
        System system;
        for (int i = 0; i < natoms; i++) system.addParticle(1.0);
        system.addForce(new RMSDForce(vec3(natoms, ref), std::vector<int>(particles, particles + n)));
        VerletIntegrator integ(0.001);
        std::map<std::string, std::string> props;
        if (precision[0]) props["Precision"] = precision;
        Context ctx(system, integ, Platform::getPlatformByName(platform), props);
        ctx.setPositions(vec3(natoms, pos));
        State s = ctx.getState(State::Energy | State::Forces);
        *energy = s.getPotentialEnergy();
        for (int i = 0; i < natoms; i++) for (int k = 0; k < 3; k++) forces[3*i + k] = s.getForces()[i][k];
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}


// A CustomCVForce of this energy expression in force group `group`, added to the System; returns its force index or -1
int rmc_add_cv_force(void* sys, const char* energy, int group) {
    try {
        CustomCVForce* f = new CustomCVForce(energy);
        f->setForceGroup(group);
        return ((System*) sys)->addForce(f);
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
static CustomCVForce& cvForce(void* sys, int index) { return dynamic_cast<CustomCVForce&>(((System*) sys)->getForce(index)); }
// collective variables of the CustomCVForce `index`: an RMSD, the distance between two group centroids (mass weights), a
// torsion plus the global `offset` (default 0) when offset is not empty, and a CustomNonbondedForce ("r", NoCutoff)
int rmc_cv_add_rmsd(void* sys, int index, const char* name, int n, const int* particles, int nref, const double* ref) {
    try { cvForce(sys, index).addCollectiveVariable(name, new RMSDForce(vec3(nref, ref), std::vector<int>(particles, particles + n))); return 0; }
    catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int rmc_cv_add_centroid_distance(void* sys, int index, const char* name, int n1, const int* g1, int n2, const int* g2, int periodic) {
    try {
        CustomCentroidBondForce* f = new CustomCentroidBondForce(2, "distance(g1,g2)");
        f->addGroup(std::vector<int>(g1, g1 + n1));
        f->addGroup(std::vector<int>(g2, g2 + n2));
        f->addBond({0, 1});
        f->setUsesPeriodicBoundaryConditions(periodic != 0);
        cvForce(sys, index).addCollectiveVariable(name, f);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int rmc_cv_add_torsion(void* sys, int index, const char* name, int a, int b, int c, int d, const char* offset) {
    try {
        CustomTorsionForce* f = new CustomTorsionForce(offset[0] ? std::string("theta+") + offset : std::string("theta"));
        if (offset[0]) f->addGlobalParameter(offset, 0.0);
        f->addTorsion(a, b, c, d);
        cvForce(sys, index).addCollectiveVariable(name, f);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int rmc_cv_add_custom_nonbonded(void* sys, int index, const char* name, int natoms) {
    try {
        CustomNonbondedForce* f = new CustomNonbondedForce("r");
        for (int i = 0; i < natoms; i++) f->addParticle({});
        cvForce(sys, index).addCollectiveVariable(name, f);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int rmc_cv_add_global(void* sys, int index, const char* name, double value, int derivative) {
    try {
        cvForce(sys, index).addGlobalParameter(name, value);
        if (derivative) cvForce(sys, index).addEnergyParameterDerivative(name);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// a Continuous2DFunction `name` of xsize x ysize values over [xmin, xmax] x [ymin, ymax]: added, or its values replaced
int rmc_cv_set_table2d(void* sys, int index, const char* name, int xsize, int ysize, const double* values, double xmin, double xmax,
                       double ymin, double ymax) {
    try {
        CustomCVForce& f = cvForce(sys, index);
        std::vector<double> v(values, values + xsize*ysize);
        for (int i = 0; i < f.getNumTabulatedFunctions(); i++)
            if (f.getTabulatedFunctionName(i) == name) {
                dynamic_cast<Continuous2DFunction&>(f.getTabulatedFunction(i)).setFunctionParameters(xsize, ysize, v, xmin, xmax, ymin, ymax);
                return 0;
            }
        f.addTabulatedFunction(name, new Continuous2DFunction(xsize, ysize, v, xmin, xmax, ymin, ymax));
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int rmc_cv_update(void* sys, int index, void* ctx) {
    try { cvForce(sys, index).updateParametersInContext(*(Context*) ctx); return 0; }
    catch (const std::exception& e) { g_err = e.what(); return -1; }
}
int rmc_cv_values(void* sys, int index, void* ctx, double* out) {
    try {
        std::vector<double> v;
        cvForce(sys, index).getCollectiveVariableValues(*(Context*) ctx, v);
        for (size_t i = 0; i < v.size(); i++) out[i] = v[i];
        return (int) v.size();
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}
// the platform a Context of this System gets when `platform` is empty, else the error of creating one on it ("" if it works)
const char* rmc_try_platform(void* sys, const char* platform) {
    static std::string out;
    try {
        VerletIntegrator integ(0.001);
        if (platform[0]) { Context ctx(*(System*) sys, integ, Platform::getPlatformByName(platform)); out = ""; }
        else { Context ctx(*(System*) sys, integ); out = ctx.getPlatform().getName(); }
    } catch (const std::exception& e) { out = std::string("error: ") + e.what(); }
    return out.c_str();
}

}
