// plugin/tests/nonbonded_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API for the parameter-change tests (tests/test_gpu_nonbonded_params.py, through oracle/omm.py Simulation): new
// base parameters of a NonbondedForce that oracle/omm_capi.cpp created, its updateParametersInContext, and a Context's
// checkpoint written to and read from a caller's buffer.  Built by plugin/Makefile (target `all`) against the
// reference's headers and oracle/_ref/libOpenMM.so.
#include "openmm/Context.h"
#include "openmm/NonbondedForce.h"
#include <cstring>
#include <exception>
#include <sstream>
#include <string>

using namespace OpenMM;

static std::string g_err;

extern "C" {

const char* nbc_last_error() { return g_err.c_str(); }

// new base parameters for the same particles and exceptions; a Context sees them after nbc_update_in_context
int nbc_set_particles(void* f, int n, const double* q, const double* sigma, const double* eps) {
    try {
        for (int k = 0; k < n; k++) ((NonbondedForce*) f)->setParticleParameters(k, q[k], sigma[k], eps[k]);
        return 0;
    } catch (std::exception& e) { g_err = e.what(); return -1; }
}
int nbc_set_exceptions(void* f, int n, const int* i, const int* j, const double* qq, const double* sigma, const double* eps) {
    try {
        for (int k = 0; k < n; k++) ((NonbondedForce*) f)->setExceptionParameters(k, i[k], j[k], qq[k], sigma[k], eps[k]);
        return 0;
    } catch (std::exception& e) { g_err = e.what(); return -1; }
}
int nbc_update_in_context(void* f, void* c) {
    try {
        ((NonbondedForce*) f)->updateParametersInContext(*(Context*) c);
        return 0;
    } catch (std::exception& e) { g_err = e.what(); return -1; }
}

// Context::createCheckpoint into buf: returns the checkpoint's size (buf NULL or cap too small: nothing copied), -1 on error
long long nbc_create_checkpoint(void* c, char* buf, long long cap) {
    try {
        std::stringstream ss(std::ios_base::in | std::ios_base::out | std::ios_base::binary);
        ((Context*) c)->createCheckpoint(ss);
        const std::string s = ss.str();
        if (buf != NULL && cap >= (long long) s.size()) memcpy(buf, s.data(), s.size());
        return (long long) s.size();
    } catch (std::exception& e) { g_err = e.what(); return -1; }
}
int nbc_load_checkpoint(void* c, const char* buf, long long size) {
    try {
        std::stringstream ss(std::string(buf, (size_t) size), std::ios_base::in | std::ios_base::binary);
        ((Context*) c)->loadCheckpoint(ss);
        return 0;
    } catch (std::exception& e) { g_err = e.what(); return -1; }
}

} // extern "C"
