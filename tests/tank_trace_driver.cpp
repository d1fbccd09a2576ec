// tank_trace_driver.cpp -- prints the C-ABI call sequence of one SPHSystem::step() of the class layer with a tank motion set.
//
// The counterpart of step_trace_driver.cpp for tests/test_cpu_tank.py: linked against host/sph_api.cpp and the generated stub of
// every sphk_* entry (each records its name and returns 0), so it runs without a device.  Each argument is one configuration
// "solver,fused,surface,vorticity,implicit,body,thresholdsNonNegative" as there; every system gets a tank motion after the
// constructor's step (a rolled tank, or with the dynamic body a shaken one: a rotating frame refuses dynamic bodies -- the python
// test's settings), and the implicit flag the constant-nu implicit viscosity (1e-3).  Prints "TRACE <configuration> <name or
// halo<what>> ..." for the step after the setting.
#include "sph_api.hpp"

#include <cstdio>
#include <string>
#include <vector>

static bool g_tracing = false;
static std::vector<std::string> g_trace;

extern "C" void step_trace_record(const char* name) {
    if (g_tracing) g_trace.emplace_back(name);
}

extern "C" int sphk_create(sphk_ctx** ctx, int, int, const sphk_grid*, void*) {
    static int dummy;
    *ctx = reinterpret_cast<sphk_ctx*>(&dummy);
    return 0;
}

static std::vector<float3> lattice(int nx, int ny, int nz, float3 origin, float spacing) {
    std::vector<float3> p;
    for (int i = 0; i < ny; ++i)
        for (int j = 0; j < nx; ++j)
            for (int k = 0; k < nz; ++k) p.push_back(make_float3(origin.x + spacing * j, origin.y + spacing * i, origin.z + spacing * k));
    return p;
}

static void traceOne(const std::string& config) {
    char solverName[16] = {0};
    int fused = 1, surface = 1, vorticity = 0, implicit = 0, body = 0, thresholds = 0;
    if (std::sscanf(config.c_str(), "%15[a-z],%d,%d,%d,%d,%d,%d", solverName, &fused, &surface, &vorticity, &implicit, &body,
                    &thresholds) != 7) {
        std::printf("bad configuration %s\n", config.c_str());
        return;
    }
    const std::string solver = solverName;
    auto fl = std::make_shared<SPHParticles>(lattice(6, 6, 6, make_float3(0.135f, 0.055f, 0.135f), 0.02f));
    auto bd = std::make_shared<SPHParticles>(lattice(4, 1, 4, make_float3(0.1f, 0.01f, 0.1f), 0.02f));
    const int n = static_cast<int>(fl->size());
    std::shared_ptr<BasicSPHSolver> basic;
    if (solver == "dfsph") basic = std::make_shared<DFSPHSolver>(n, thresholds ? 1e-3f : -1.0f, thresholds ? 1e-3f : -1.0f, 4);
    else if (solver == "pbd") basic = std::make_shared<PBDSolver>(n, 4);
    else basic = std::make_shared<BasicSPHSolver>(n);
    basic->setFusedSweeps(fused != 0);
    if (vorticity) basic->setVorticityConfinement(0.2f);
    if (implicit) basic->setImplicitViscosity(1e-3f);
    basic->setFieldHook([](int what, float*, int) {
        if (g_tracing) g_trace.push_back("halo" + std::to_string(what));
    });
    std::vector<sphb200::KinematicBody> bodies;
    if (body) {
        sphb200::KinematicBody b;
        b.points = lattice(2, 2, 2, make_float3(-0.01f, -0.01f, -0.01f), 0.02f);
        b.position = make_float3(0.25f, 0.35f, 0.25f);
        b.orientation = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
        b.linearVelocity = make_float3(0.0f, 0.0f, 0.0f);
        b.angularVelocity = make_float3(0.0f, 0.0f, 0.0f);
        b.mass = 1e-3f;
        b.inertia = make_float3(1e-7f, 1e-7f, 1e-7f);
        bodies.push_back(b);
    }
    std::shared_ptr<BaseSolver> s = basic;
    const float st = surface ? 1e-4f : 0.0f;
    SPHSystem sys(fl, bd, s, make_float3(0.5f, 0.5f, 0.5f), 0.0404f, 0.04f, solver == "wcsph" ? 0.001f : 0.004f, 76.596750762082e-6f,
                  1.0f, 1.4f, 10.0f, 5e-4f, st, st, make_float3(0.0f, -9.8f, 0.0f), make_int3(13, 13, 13), bodies);
    sys.setStepGraph(false);
    sphb200::TankMotion m;
    if (body) {
        sphb200::TankHarmonic h;
        h.amplitude = make_float3(2.0f, 0.0f, 0.0f);
        h.omega = 6.0f;
        m.harmonics.push_back(h);
    } else {
        m.axis = make_float3(0.0f, 0.0f, 1.0f);
        m.pivot = make_float3(0.25f, 0.0f, 0.25f);
        m.rollAmplitude = 0.1f;
        m.rollOmega = 4.0f;
        m.ramp = 0.5f;
    }
    if (!sys.setTankMotion(m)) {
        std::printf("setTankMotion refused\n");
        return;
    }
    g_trace.clear();
    g_tracing = true;
    sys.step();
    g_tracing = false;
    std::string line = "TRACE " + config;
    for (const auto& t : g_trace) line += " " + t;
    std::printf("%s\n", line.c_str());
}

int main(int argc, char** argv) {
    for (int a = 1; a < argc; ++a) traceOne(argv[a]);
    return 0;
}
