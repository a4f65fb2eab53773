// plugin/tests/bonded_objects.cpp -- two Force objects of every bonded class on the B200 platform, against the Reference
// platform in the same process.
//
// Each class gets a System with two objects: object 1 in force group 1, object 2 in force group 2 with periodic boundary
// conditions in a large box.  The terms of object 2 follow those of object 1 in the platform's per-class arrays, so every
// update of object 2 writes a range that does not start at term 0.  Per-group and total forces and energies are compared
// at the start, after updateParametersInContext of object 2 alone, then of object 1 alone (CMAP: a term also changes its
// map; custom torsions: then a global parameter changes too); finally a changed atom of object 2 must be refused.
// Tolerances are those of the reference's own test bodies (tests/Test<X>.h).  Built by plugin/Makefile (target
// `reftests`); B200_PLUGIN names the plugin library.
#include "openmm/Context.h"
#include "openmm/Platform.h"
#include "openmm/State.h"
#include "openmm/System.h"
#include "openmm/VerletIntegrator.h"
#include "openmm/HarmonicBondForce.h"
#include "openmm/HarmonicAngleForce.h"
#include "openmm/PeriodicTorsionForce.h"
#include "openmm/RBTorsionForce.h"
#include "openmm/CMAPTorsionForce.h"
#include "openmm/CustomTorsionForce.h"
#include "openmm/OpenMMException.h"
#include "openmm/internal/AssertionUtilities.h"
#include <cmath>
#include <cstdlib>
#include <iostream>
#include <string>
#include <vector>

using namespace OpenMM;
using namespace std;

const double TOL = 1e-5;

// a non-degenerate chain of ten atoms, every coordinate a multiple of 1/32 nm (exact in fp32)
const double POS[10][3] = {{1.0, 1.0, 1.0}, {0.84375, 1.09375, 0.9375}, {0.8125, 1.15625, 1.03125}, {0.84375, 1.3125, 0.9375},
                           {0.71875, 1.28125, 1.0}, {0.71875, 1.125, 1.0}, {0.78125, 1.15625, 0.84375}, {0.90625, 1.21875, 0.8125},
                           {0.75, 1.28125, 0.78125}, {0.84375, 1.40625, 0.84375}};

Platform* b200;

void compare(const string& what, Context& a, Context& ref, double ftol, double etol) {
    for (int groups : {1 << 1, 1 << 2, -1}) {
        const State s = a.getState(State::Forces | State::Energy, false, groups);
        const State r = ref.getState(State::Forces | State::Energy, false, groups);
        try {
            for (size_t i = 0; i < r.getForces().size(); i++) ASSERT_EQUAL_VEC(r.getForces()[i], s.getForces()[i], ftol);
            ASSERT_EQUAL_TOL(r.getPotentialEnergy(), s.getPotentialEnergy(), etol);
        } catch (const exception& e) {
            throw OpenMMException(what + ", groups " + to_string(groups) + ": " + e.what());
        }
    }
}

// change(force, obj) gives object obj new parameters; moveAtom(force) changes an atom of its first term
template<class F, class Change, class Move>
void run(const string& name, F* f1, F* f2, Change change, Move moveAtom, double ftol = TOL, double etol = TOL, const string& global = "") {
    cout << "[run] " << name << endl;
    System system;
    vector<Vec3> pos;
    for (int i = 0; i < 10; i++) { system.addParticle(1.0); pos.push_back(Vec3(POS[i][0], POS[i][1], POS[i][2])); }
    system.setDefaultPeriodicBoxVectors(Vec3(10, 0, 0), Vec3(0, 10, 0), Vec3(0, 0, 10));
    f1->setForceGroup(1);
    f2->setForceGroup(2);
    f2->setUsesPeriodicBoundaryConditions(true);
    system.addForce(f1);
    system.addForce(f2);
    VerletIntegrator i1(0.001), i2(0.001);
    Context a(system, i1, *b200), ref(system, i2, Platform::getPlatformByName("Reference"));
    a.setPositions(pos);
    ref.setPositions(pos);
    compare(name + " initial", a, ref, ftol, etol);
    change(*f2, 2);
    f2->updateParametersInContext(a);
    f2->updateParametersInContext(ref);
    compare(name + " after updating object 2", a, ref, ftol, etol);
    change(*f1, 1);
    f1->updateParametersInContext(a);
    f1->updateParametersInContext(ref);
    compare(name + " after updating object 1", a, ref, ftol, etol);
    if (!global.empty()) {
        a.setParameter(global, 2.5);
        ref.setParameter(global, 2.5);
        compare(name + " after setting " + global, a, ref, ftol, etol);
    }
    moveAtom(*f2);
    try {
        f2->updateParametersInContext(a);
    } catch (const OpenMMException& e) {
        if (string(e.what()).find("The set of particles in") != string::npos) return;
        throw OpenMMException(name + ": a changed atom of object 2 was refused with '" + e.what() + "'");
    }
    throw OpenMMException(name + ": a changed atom of object 2 was accepted");
}

// a smooth periodic map of size n
vector<double> cmapEnergy(int n, double amp, double shift) {
    vector<double> e(n*n);
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) e[i + n*j] = amp*(cos(2*M_PI*i/n + shift) + 0.5*sin(2*M_PI*j/n - shift));
    return e;
}

int main() {
    try {
        const char* path = getenv("B200_PLUGIN");
        Platform::loadPluginLibrary(path ? path : "libOpenMMB200.so");
        b200 = &Platform::getPlatformByName("B200");

        HarmonicBondForce* b1 = new HarmonicBondForce(), *b2 = new HarmonicBondForce();
        b1->addBond(0, 1, 0.12, 300.0); b1->addBond(1, 2, 0.14, 250.0); b1->addBond(2, 3, 0.15, 200.0);
        b2->addBond(3, 4, 0.13, 350.0); b2->addBond(5, 6, 0.16, 280.0); b2->addBond(7, 8, 0.11, 320.0);
        run("HarmonicBondForce", b1, b2,
            [](HarmonicBondForce& f, int obj) {
                for (int t = 0; t < f.getNumBonds(); t++) {
                    int p, q; double r0, k;
                    f.getBondParameters(t, p, q, r0, k);
                    f.setBondParameters(t, p, q, r0 + 0.01*obj, k*(1.5 + 0.25*t));
                }
            },
            [](HarmonicBondForce& f) { f.setBondParameters(0, 3, 5, 0.13, 350.0); });

        HarmonicAngleForce* a1 = new HarmonicAngleForce(), *a2 = new HarmonicAngleForce();
        a1->addAngle(0, 1, 2, 1.9, 80.0); a1->addAngle(1, 2, 3, 2.0, 90.0);
        a2->addAngle(3, 4, 5, 1.8, 100.0); a2->addAngle(5, 6, 7, 2.1, 70.0); a2->addAngle(6, 7, 8, 1.7, 110.0);
        run("HarmonicAngleForce", a1, a2,
            [](HarmonicAngleForce& f, int obj) {
                for (int t = 0; t < f.getNumAngles(); t++) {
                    int p, q, r; double theta, k;
                    f.getAngleParameters(t, p, q, r, theta, k);
                    f.setAngleParameters(t, p, q, r, theta - 0.1*obj, k*(1.5 + 0.25*t));
                }
            },
            [](HarmonicAngleForce& f) { f.setAngleParameters(0, 3, 4, 6, 1.8, 100.0); });

        PeriodicTorsionForce* t1 = new PeriodicTorsionForce(), *t2 = new PeriodicTorsionForce();
        t1->addTorsion(0, 1, 2, 3, 1, 0.5, 5.0); t1->addTorsion(1, 2, 3, 4, 2, 1.0, 3.0);
        t2->addTorsion(3, 4, 5, 6, 3, 0.0, 4.0); t2->addTorsion(5, 6, 7, 8, 1, 2.0, 6.0); t2->addTorsion(6, 7, 8, 9, 2, -1.0, 2.0);
        run("PeriodicTorsionForce", t1, t2,
            [](PeriodicTorsionForce& f, int obj) {
                for (int t = 0; t < f.getNumTorsions(); t++) {
                    int p, q, r, s, n; double phase, k;
                    f.getTorsionParameters(t, p, q, r, s, n, phase, k);
                    f.setTorsionParameters(t, p, q, r, s, n + obj, phase + 0.3, k*(1.5 + 0.25*t));
                }
            },
            [](PeriodicTorsionForce& f) { f.setTorsionParameters(0, 3, 4, 5, 7, 3, 0.0, 4.0); });

        RBTorsionForce* r1 = new RBTorsionForce(), *r2 = new RBTorsionForce();
        r1->addTorsion(0, 1, 2, 3, 1.0, 2.0, -1.5, 0.5, 0.25, -0.1); r1->addTorsion(1, 2, 3, 4, 0.5, -1.0, 2.0, 1.0, -0.5, 0.2);
        r2->addTorsion(3, 4, 5, 6, 2.0, 1.0, 0.5, -1.0, 0.3, 0.1); r2->addTorsion(5, 6, 7, 8, -1.0, 0.5, 1.5, 0.2, -0.2, 0.4);
        r2->addTorsion(6, 7, 8, 9, 0.3, -0.7, 1.1, -0.4, 0.6, -0.3);
        run("RBTorsionForce", r1, r2,
            [](RBTorsionForce& f, int obj) {
                for (int t = 0; t < f.getNumTorsions(); t++) {
                    int p, q, r, s; double c[6];
                    f.getTorsionParameters(t, p, q, r, s, c[0], c[1], c[2], c[3], c[4], c[5]);
                    for (int k = 0; k < 6; k++) c[k] = 0.5*c[k] + 0.1*(k + obj + t);
                    f.setTorsionParameters(t, p, q, r, s, c[0], c[1], c[2], c[3], c[4], c[5]);
                }
            },
            [](RBTorsionForce& f) { f.setTorsionParameters(0, 3, 4, 5, 7, 2.0, 1.0, 0.5, -1.0, 0.3, 0.1); });

        // object 1: one map, one term; object 2: two maps, two terms (the update swaps their maps)
        CMAPTorsionForce* c1 = new CMAPTorsionForce(), *c2 = new CMAPTorsionForce();
        c1->addMap(12, cmapEnergy(12, 8.0, 0.3));
        c1->addTorsion(0, 0, 1, 2, 3, 1, 2, 3, 4);
        c2->addMap(10, cmapEnergy(10, 5.0, 1.1));
        c2->addMap(16, cmapEnergy(16, 12.0, -0.7));
        c2->addTorsion(0, 3, 4, 5, 6, 4, 5, 6, 7);
        c2->addTorsion(1, 5, 6, 7, 8, 6, 7, 8, 9);
        run("CMAPTorsionForce", c1, c2,
            [](CMAPTorsionForce& f, int obj) {
                for (int m = 0; m < f.getNumMaps(); m++) {
                    int n; vector<double> e;
                    f.getMapParameters(m, n, e);
                    f.setMapParameters(m, n, cmapEnergy(n, 3.0 + 4*m, 0.5*obj));
                }
                for (int t = 0; t < f.getNumTorsions(); t++) {
                    int map, a[8];
                    f.getTorsionParameters(t, map, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);
                    f.setTorsionParameters(t, f.getNumMaps() - 1 - map, a[0], a[1], a[2], a[3], a[4], a[5], a[6], a[7]);
                }
            },
            [](CMAPTorsionForce& f) { f.setTorsionParameters(0, 1, 3, 4, 5, 6, 4, 5, 6, 8); }, 0.05, 1e-3);

        // different expressions and numbers of per-torsion parameters; object 2 reads a global parameter
        CustomTorsionForce* u1 = new CustomTorsionForce("k*(1+cos(n*theta-theta0))"), *u2 = new CustomTorsionForce("scale*k*(theta-t0)^2");
        u1->addPerTorsionParameter("k"); u1->addPerTorsionParameter("n"); u1->addPerTorsionParameter("theta0");
        u2->addPerTorsionParameter("k"); u2->addPerTorsionParameter("t0"); u2->addGlobalParameter("scale", 1.0);
        u1->addTorsion(0, 1, 2, 3, {5.0, 1, 0.5}); u1->addTorsion(1, 2, 3, 4, {3.0, 2, 1.0});
        u2->addTorsion(3, 4, 5, 6, {4.0, -0.5}); u2->addTorsion(5, 6, 7, 8, {6.0, 1.0}); u2->addTorsion(6, 7, 8, 9, {2.0, 2.5});
        run("CustomTorsionForce", u1, u2,
            [](CustomTorsionForce& f, int obj) {
                for (int t = 0; t < f.getNumTorsions(); t++) {
                    int p, q, r, s; vector<double> par;
                    f.getTorsionParameters(t, p, q, r, s, par);
                    par[0] *= 1.5 + 0.25*t;
                    par[1] += 0.2*obj;
                    f.setTorsionParameters(t, p, q, r, s, par);
                }
            },
            [](CustomTorsionForce& f) { f.setTorsionParameters(0, 3, 4, 5, 7, {4.0, -0.5}); }, TOL, TOL, "scale");
    } catch (const exception& e) {
        cout << "exception: " << e.what() << endl;
        return 1;
    }
    cout << "Done" << endl;
    return 0;
}
