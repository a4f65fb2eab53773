// plugin/tests/gbsa_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the ctypes harness of the generalized Born tests (tests/gbsa_harness.py): the reference's public
// GBSAOBCForce, added to a System that oracle/omm_capi.cpp created, and its updateParametersInContext.
// Built by plugin/Makefile (target `reftests`) against the reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/GBSAOBCForce.h"
#include "openmm/VerletIntegrator.h"
#include <exception>
#include <string>

using namespace OpenMM;

static std::string g_err;

extern "C" {

const char* gbc_last_error() { return g_err.c_str(); }

// A GBSAOBCForce with these per-particle parameters, method (GBSAOBCForce::NonbondedMethod), cutoff, dielectrics and surface
// energy, in force group `group`, added to the System; returns its force index or -1
int gbc_add_force(void* sys, int n, const double* q, const double* radius, const double* scale, int method, double cutoff,
                  double solute, double solvent, double surface, int group) {
    try {
        GBSAOBCForce* f = new GBSAOBCForce();
        for (int i = 0; i < n; i++) f->addParticle(q[i], radius[i], scale[i]);
        f->setNonbondedMethod((GBSAOBCForce::NonbondedMethod) method);
        f->setCutoffDistance(cutoff);
        f->setSoluteDielectric(solute);
        f->setSolventDielectric(solvent);
        f->setSurfaceAreaEnergy(surface);
        f->setForceGroup(group);
        return ((System*) sys)->addForce(f);
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// New parameters for the first n particles of force `index` (n may differ from its count: the force then grows or keeps its
// count as given), then updateParametersInContext
int gbc_update(void* sys, int index, void* ctx, int n, const double* q, const double* radius, const double* scale) {
    try {
        GBSAOBCForce& f = dynamic_cast<GBSAOBCForce&>(((System*) sys)->getForce(index));
        for (int i = 0; i < n; i++) {
            if (i < f.getNumParticles()) f.setParticleParameters(i, q[i], radius[i], scale[i]);
            else f.addParticle(q[i], radius[i], scale[i]);
        }
        f.updateParametersInContext(*(Context*) ctx);
        return 0;
    } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// The platform a Context of this System gets when none is named ("" on failure)
const char* gbc_default_platform(void* sys) {
    static std::string name;
    try {
        VerletIntegrator integ(0.001);
        Context ctx(*(System*) sys, integ);
        name = ctx.getPlatform().getName();
    } catch (const std::exception& e) { g_err = e.what(); name = ""; }
    return name.c_str();
}

}
