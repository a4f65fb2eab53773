// plugin/tests/cmap_rb_capi.cpp -- TEST INFRASTRUCTURE, not product code.
//
// A flat C API over the reference's public RBTorsionForce and CMAPTorsionForce, for the ctypes harness of the RB / CMAP tests
// (tests/cmap_rb_harness.py).  It adds those forces to a System that oracle/omm_capi.cpp created, and exposes the
// reference's own CMAP spline fitter.  Built by plugin/Makefile (target `reftests`) against the staged headers and
// oracle/_ref/libOpenMM.so.
#include "openmm/System.h"
#include "openmm/RBTorsionForce.h"
#include "openmm/CMAPTorsionForce.h"
#include "openmm/internal/CMAPTorsionForceImpl.h"
#include <vector>

using namespace OpenMM;

extern "C" {

// c: [n][6]; returns the index of the force in the System
int cmap_rb_add_rb_torsions(void* system, int n, const int* i, const int* j, const int* k, const int* l, const double* c, int periodic, int group) {
    RBTorsionForce* f = new RBTorsionForce();
    for (int t = 0; t < n; t++) f->addTorsion(i[t], j[t], k[t], l[t], c[6*t], c[6*t+1], c[6*t+2], c[6*t+3], c[6*t+4], c[6*t+5]);
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// energy: the maps one after the other, size[m]^2 values each (CMAPTorsionForce::addMap); atoms: [n][8]
int cmap_rb_add_cmap(void* system, int nmaps, const int* size, const double* energy, int n, const int* map, const int* atoms, int periodic, int group) {
    CMAPTorsionForce* f = new CMAPTorsionForce();
    for (int m = 0; m < nmaps; m++) {
        f->addMap(size[m], std::vector<double>(energy, energy + size[m]*size[m]));
        energy += size[m]*size[m];
    }
    for (int t = 0; t < n; t++) {
        const int* a = atoms + 8*t;
        f->addTorsion(map[t], a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);
    }
    f->setUsesPeriodicBoundaryConditions(periodic != 0);
    f->setForceGroup(group);
    return ((System*) system)->addForce(f);
}

// CMAPTorsionForceImpl::calcMapDerivatives: the bicubic coefficients of one map, out [size^2][16]
void cmap_rb_coefficients(int size, const double* energy, double* out) {
    std::vector<std::vector<double> > c;
    CMAPTorsionForceImpl::calcMapDerivatives(size, std::vector<double>(energy, energy + size*size), c);
    for (int p = 0; p < size*size; p++) for (int k = 0; k < 16; k++) out[16*p+k] = c[p][k];
}

} // extern "C"
