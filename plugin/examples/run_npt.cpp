// run_npt.cpp -- a C++ host application for constant-pressure runs: a System from XML (XmlSerializer::deserialize<System>)
// plus a MonteCarloBarostat or MonteCarloAnisotropicBarostat, on any platform, through the reference's public API only.
// The reference's own MonteCarloBarostatImpl drives the platform's ApplyMonteCarloBarostatKernel.
//
//   run_npt system.xml positions.f64 out.bin [--platform B200] [--plugin plugin/libOpenMMB200.so] [--device 0]
//           [--integrator langevin_middle|verlet] [--dt 0.002] [--temperature 300] [--friction 1] [--seed 7]
//           [--barostat 1] [--pressure 1] [--frequency 25] [--barostat-seed 1] [--warmup 0] [--chunks 1] [--chunk-steps 1000]
//
// positions.f64: the coordinates as 3N little-endian doubles (nm).  --barostat: 0 none, 1 MonteCarloBarostat, 2
// MonteCarloAnisotropicBarostat scaling x, y and z.  Velocities: Context::setVelocitiesToTemperature(temperature, 11) with the
// Langevin integrator, zero with Verlet (--temperature is then the barostat's alone).  After `warmup` untimed steps, out.bin receives Context::getMolecules() (int32 nmol,
// int32 start[nmol+1], int32 atoms[start[nmol]]) and then, for the initial state and after each of `chunks` runs of
// `chunk-steps` steps, the box (9 doubles, rows a, b, c) and the positions (3N doubles).  Prints one JSON line with the
// ns/day of the chunks (state reads included) and the volume at the start and at the end.
#include "openmm/Platform.h"
#include "openmm/System.h"
#include "openmm/Context.h"
#include "openmm/State.h"
#include "openmm/LangevinMiddleIntegrator.h"
#include "openmm/VerletIntegrator.h"
#include "openmm/MonteCarloBarostat.h"
#include "openmm/MonteCarloAnisotropicBarostat.h"
#include "openmm/OpenMMException.h"
#include "openmm/serialization/XmlSerializer.h"
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <map>
#include <memory>
#include <string>
#include <vector>

using namespace OpenMM;

static void writeFrame(std::ofstream& out, const State& st) {
    Vec3 box[3];
    st.getPeriodicBoxVectors(box[0], box[1], box[2]);
    for (int i = 0; i < 3; i++) { const double v[3] = {box[i][0], box[i][1], box[i][2]}; out.write((const char*) v, sizeof(v)); }
    for (const Vec3& p : st.getPositions()) { const double v[3] = {p[0], p[1], p[2]}; out.write((const char*) v, sizeof(v)); }
}

static double volume(const State& st) {
    Vec3 a, b, c;
    st.getPeriodicBoxVectors(a, b, c);
    return a[0]*b[1]*c[2];
}

int main(int argc, char** argv) {
    if (argc < 4) { fprintf(stderr, "usage: %s system.xml positions.f64 out.bin [--option value ...] (see the header of run_npt.cpp)\n", argv[0]); return 2; }
    std::map<std::string, std::string> opt = {{"--platform", "B200"}, {"--plugin", "plugin/libOpenMMB200.so"}, {"--device", "0"},
                                              {"--integrator", "langevin_middle"}, {"--dt", "0.002"}, {"--temperature", "300"}, {"--friction", "1"},
                                              {"--seed", "7"}, {"--barostat", "1"}, {"--pressure", "1"}, {"--frequency", "25"}, {"--barostat-seed", "1"},
                                              {"--warmup", "0"}, {"--chunks", "1"}, {"--chunk-steps", "1000"}};
    for (int i = 4; i + 1 < argc; i += 2) {
        if (!opt.count(argv[i])) { fprintf(stderr, "unknown option %s\n", argv[i]); return 2; }
        opt[argv[i]] = argv[i+1];
    }
    try {
        std::ifstream xml(argv[1]);
        if (!xml) throw OpenMMException(std::string("cannot open ") + argv[1]);
        std::unique_ptr<System> system(XmlSerializer::deserialize<System>(xml));
        const int n = system->getNumParticles();
        std::ifstream pin(argv[2], std::ios::binary);
        std::vector<double> raw(3*(size_t) n);
        if (!pin.read((char*) raw.data(), raw.size()*sizeof(double))) throw OpenMMException(std::string("cannot read 3N doubles from ") + argv[2]);
        std::vector<Vec3> positions(n);
        for (int i = 0; i < n; i++) positions[i] = Vec3(raw[3*i], raw[3*i+1], raw[3*i+2]);

        const double pressure = atof(opt["--pressure"].c_str()), temperature = atof(opt["--temperature"].c_str());
        const int frequency = atoi(opt["--frequency"].c_str()), kind = atoi(opt["--barostat"].c_str());
        if (kind == 1) {
            MonteCarloBarostat* b = new MonteCarloBarostat(pressure, temperature, frequency);
            b->setRandomNumberSeed(atoi(opt["--barostat-seed"].c_str()));
            system->addForce(b);
        }
        else if (kind == 2) {
            MonteCarloAnisotropicBarostat* b = new MonteCarloAnisotropicBarostat(Vec3(pressure, pressure, pressure), temperature, true, true, true, frequency);
            b->setRandomNumberSeed(atoi(opt["--barostat-seed"].c_str()));
            system->addForce(b);
        }
        else if (kind != 0) throw OpenMMException("--barostat must be 0, 1 or 2");

        const double dt = atof(opt["--dt"].c_str());
        std::unique_ptr<Integrator> integrator;
        if (opt["--integrator"] == "verlet") integrator.reset(new VerletIntegrator(dt));
        else if (opt["--integrator"] == "langevin_middle") {
            LangevinMiddleIntegrator* li = new LangevinMiddleIntegrator(temperature, atof(opt["--friction"].c_str()), dt);
            li->setRandomNumberSeed(atoi(opt["--seed"].c_str()));
            integrator.reset(li);
        }
        else throw OpenMMException("--integrator must be langevin_middle or verlet");

        if (opt["--platform"] == "B200") Platform::loadPluginLibrary(opt["--plugin"]);
        Platform& platform = Platform::getPlatformByName(opt["--platform"]);
        std::map<std::string, std::string> props;
        if (opt["--platform"] == "B200") props["DeviceIndex"] = opt["--device"];
        Context context(*system, *integrator, platform, props);
        context.setPositions(positions);
        if (opt["--integrator"] != "verlet") context.setVelocitiesToTemperature(temperature, 11);
        integrator->step(atoi(opt["--warmup"].c_str()));

        std::ofstream out(argv[3], std::ios::binary);
        const std::vector<std::vector<int> >& mols = context.getMolecules();
        const int nmol = (int) mols.size();
        std::vector<int> start(1, 0), atoms;
        for (const std::vector<int>& m : mols) { atoms.insert(atoms.end(), m.begin(), m.end()); start.push_back((int) atoms.size()); }
        out.write((const char*) &nmol, sizeof(int));
        out.write((const char*) start.data(), start.size()*sizeof(int));
        out.write((const char*) atoms.data(), atoms.size()*sizeof(int));
        const State s0 = context.getState(State::Positions);
        writeFrame(out, s0);

        const int chunks = atoi(opt["--chunks"].c_str()), chunkSteps = atoi(opt["--chunk-steps"].c_str());
        double volEnd = volume(s0);
        const auto t0 = std::chrono::steady_clock::now();
        for (int k = 0; k < chunks; k++) {
            integrator->step(chunkSteps);
            const State st = context.getState(State::Positions);      // drains the device
            writeFrame(out, st);
            volEnd = volume(st);
        }
        const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
        const long steps = (long) chunks*chunkSteps;
        printf("{\"atoms\": %d, \"platform\": \"%s\", \"barostat\": %d, \"frequency\": %d, \"steps\": %ld, \"dt_fs\": %.3f, \"ns_per_day\": %.2f, "
               "\"volume_start\": %.6f, \"volume_end\": %.6f, \"molecules\": %d}\n", n, context.getPlatform().getName().c_str(), kind, frequency, steps,
               1e3*dt, sec > 0 ? dt*1e-3*steps*86400.0/sec : 0.0, volume(s0), volEnd, nmol);
    }
    catch (const std::exception& e) {
        fprintf(stderr, "run_npt: %s\n", e.what());
        return 1;
    }
    return 0;
}
