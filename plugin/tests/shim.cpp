// plugin/tests/shim.cpp -- runs the REFERENCE'S OWN platform-parametrised test bodies (tests/Test<X>.h, read where
// they lie under /root/reference, never copied) against the B200 platform, the way platforms/cuda/tests/CudaTests.h:38-43
// + TestCuda<X>.cpp do for the CUDA platform.  Built by plugin/Makefile (target `reftests`) with
//   -DTEST_HEADER="\"TestEwald.h\"" -DTEST_CALLS="testTriclinic(); testPMEParameters();"
// The reference header's own main() is renamed away; TEST_CALLS lists the test functions whose features the B200
// platform implements (plugin/Makefile has the list per header; not called: Ewald summation, LJPME, two NonbondedForce
// objects, virtual sites and everything that needs a Custom*Force -- outside the hot path, SURVEY.md section 8).
#include "openmm/Platform.h"
#include "openmm/OpenMMException.h"
#include <cstdlib>
#include <iostream>
#include <string>

// -DB200_PRECISION='"mixed"' runs the same bodies with that Precision as the platform default, as
// platforms/cuda/tests/CudaTests.h does with its precision argument
static OpenMM::Platform& loadB200() {
    const char* path = getenv("B200_PLUGIN");
    OpenMM::Platform::loadPluginLibrary(path ? path : "libOpenMMB200.so");
    OpenMM::Platform& p = OpenMM::Platform::getPlatformByName("B200");
#ifdef B200_PRECISION
    p.setPropertyDefaultValue("Precision", B200_PRECISION);
#endif
    return p;
}
OpenMM::Platform& platform = loadB200();

void initializeTests(int argc, char* argv[]) {
}

#define main reference_main_unused
#include TEST_HEADER
#undef main

void runPlatformTests() {
}

#define T(x) do { std::cout << "[run] " #x << std::endl; x; } while (0)

int main(int argc, char* argv[]) {
    try {
        TEST_CALLS
    }
    catch (const std::exception& e) {
        std::cout << "exception: " << e.what() << std::endl;
        return 1;
    }
    std::cout << "Done" << std::endl;
    return 0;
}
