// sph_headless.cpp -- the reference application without its window (SURVEY 8f-1).
//
// What main.cpp does around the hot path, and nothing else: build the dam-break scene (constants main.cpp:54-67,
// fluid block :75-86, boundary shell :89-117), pick a solver (:119-130), construct SPHSystem (:131-134), then call
// step() per frame and print the reference's timing line (oneStep, :300-306).  Written against the class API only
// (SPHSystem / SPHParticles / *Solver, the names the reference exports), so the same call sites run on this engine.
// Additions: scene size and solver settings from the command line, a JSON summary, an optional particle dump
// (positions, densities and the generate_dots colours of vbo.cu:26-51) for offline viewing.
//
//   sph_headless [--solver sph|dfsph|pbd] [--frames N] [--box L | --box LX LY LZ] [--block NX NY NZ] [--origin X Y Z]
//                [--dt DT] [--iters K] [--vorticity EPS] [--dump PREFIX] [--quiet] [--emit-scene PREFIX] [--ranks N [--rank R --rendezvous DIR]]
//                [--bullets K] [--stir OMEGA] [--float REL] [--implicit-viscosity NU] [--tap SPEED] [--drain SIDE] [--capacity N]
//                [--cfl C [--dt-min X]] [--rheology cross:NU0,NUINF,LAMBDA,M | hb:K,N,TAU[,MREG] [--rheology-max NU_MAX] [--no-slip]]
//                [--heat ALPHA,BETA[,TREF] [--heater T] [--wall-temp T[,H]] [--tap-temp T] [--thermal-viscosity NUREF,E[,NUMAX]]]
//                [--adhesion BETA[,BODYBETA]] [--obstacle FILE[,S,X,Y,Z]]... [--mesh-body FILE,REL[,S,X,Y,Z]] [--fluid-mesh FILE[,S,X,Y,Z]]
//                [--probe X,Y,Z]... [--gauge AX,AY,AZ,BX,BY,BZ[,K]]... [--gauge-threshold THETA] [--probe-out FILE]
//                [--tank-roll DEG,HZ[,PX,PY,PZ,NX,NY,NZ]] [--tank-shake AX,AY,AZ,HZ] [--tank-accel AX,AY,AZ] [--tank-spin RAD_S]
//                [--tank-ramp SEC]
// --tank-roll, --tank-shake, --tank-accel and --tank-spin move the tank (SPHSystem::setTankMotion, DESIGN.md section 2.15) from the
// step after the constructor's step 0 on; the simulation runs in the tank's frame, so every output (dump, probes, gauges) is in tank
// coordinates.  --tank-roll rolls it by DEG degrees at HZ about the axis N through the pivot P (default: the z axis through the
// bottom centre (L/2, 0, L/2)); --tank-spin spins it at RAD_S about the roll's axis, or without --tank-roll about the vertical axis
// through the bottom centre; --tank-shake shakes it with the world acceleration (AX, AY, AZ) sin(2 pi HZ t) (m/s^2), --tank-accel
// adds a constant one; --tank-ramp ramps all of it in over SEC seconds.  Every frame prints theta and a_w.  Single GPU only; not
// with --heat.
// --probe and --gauge (repeatable; DESIGN.md section 2.13) record SPH-interpolated fields at points and water levels along segments
// every step after the constructor's step 0 (SPHSystem::setProbes): a gauge runs from A to B with K samples (default 64), its
// level is its height above A (orient it upwards, along -G, from the floor), wet where the Shepard sum reaches THETA (default 0.5).
// --probe-out FILE (required with them) gets a CSV row per step: step,t, then each probe's S,rho,vx,vy,vz,p,T,n, then each gauge's
// level (-1: dry).  The device ring is drained after every frame (sized for a frame's largest substep count with --cfl).  At most
// 4096 probes and 64 gauges; single GPU only.
// --checkpoint FILE [--checkpoint-every K] saves the state (SPHSystem::checkpoint, DESIGN.md section 2.14) after every K-th frame
// (K = 0, the default: none before the last) and after the last frame; the file is written behind the following frames.
// --resume FILE restores such a file into the system the same scene and setting flags build and continues from its frame to
// --frames; with --probe-out the rows of the resumed frames are appended to the CSV.  Single GPU only; not with --bullets.
// --obstacle, --mesh-body and --fluid-mesh build the scene from Wavefront OBJ meshes (sphb200::loadObj, DESIGN.md section 2.12), each
// mapped by S * v + (X, Y, Z) (default 1 and 0).  --obstacle (repeatable) is a static obstacle: its surface sampled at the boundary
// spacing (sphb200::sampleSurface) is appended to the boundary set after the tank shell, so it has the walls' adhesion and
// temperature.  --mesh-body adds one body (sphb200::meshBody) of relative density REL (0: kinematic, at rest), not together with
// --stir, --float or --heater; with it the result line carries the body's pose, motion and last impulse.  --fluid-mesh fills the
// mesh at the fluid spacing from --origin (sphb200::fillMesh) instead of the block.  The fluid is cleared of every obstacle and the
// body at the boundary spacing (sphb200::clearOf), which needs the inside of every mesh: all three options take closed meshes
// only, and every mesh must lie in [0, 0.99 box].  Single GPU only; with them --emit-scene needs a GPU too.
// --adhesion turns on fluid-solid adhesion (BasicSPHSolver::setAdhesion, DESIGN.md section 2.11) after the constructor's step 0: the
// tank walls with BETA, the --stir paddle, the --float cube or the --heater plate with BODYBETA (default BETA).  Every frame prints
// the wetted particles and the largest adhesion acceleration; with --float the result line also carries the cube's position and its
// last step's impulse.  Single GPU only.
// --heat turns on heat transfer (BasicSPHSolver::setThermal, DESIGN.md section 2.10) after the constructor's step 0: diffusivity ALPHA,
// buoyancy BETA, reference temperature TREF (default 0, also the fluid's initial temperature).  --heater T adds a held, motionless
// plate body on the floor under the block at T with conductance 1 (not together with --stir or --float); --wall-temp T[,H] sets the
// tank walls' temperature and conductance (default TREF, 0: adiabatic); --tap-temp T the --tap emitter's temperature (default TREF).
// --thermal-viscosity NUREF,E[,NUMAX] solves nu = clamp(NUREF exp(-E (T - TREF)), 0, NUMAX) (default NUMAX = 100 NUREF) with no-slip
// walls instead of a constant nu (not with --rheology, --implicit-viscosity or --float).  Every frame prints min, max and mean T, the
// heat content sum m T, the substeps and the particle-substeps above the stability bound.  Single GPU only.
// --rheology turns on non-Newtonian viscosity (BasicSPHSolver::setRheology, DESIGN.md section 2.9) after the constructor's step 0,
// for every solver, instead of --implicit-viscosity: a Cross fluid (shear-thinning; Newtonian with NU0 = NUINF) or a
// Herschel-Bulkley fluid with yield stress TAU (kinematic; Bingham with N = 1), regularisation MREG (default 1000 s).  nu is
// clamped to [0, NU_MAX]; NU_MAX defaults to max(NU0, NUINF) for Cross and to 1 for Herschel-Bulkley.  --no-slip: walls and a
// --stir paddle act with the fluid's own nu (boundary factor 1; default 0, free slip; not together with --float).  Every frame
// prints the solve's iterations, the largest shear rate and the particles at the NU_MAX clamp.  Single GPU only.
// --cfl C turns on CFL-adaptive time stepping (SPHSystem::setAdaptiveTimeStep, DESIGN.md section 2.8) after the constructor's step 0:
// every frame then advances --dt of simulated time in CFL substeps (SPHSystem::advance; dt_max = --dt, dt_min = X or dt / 64) and
// prints their count and the smallest dt of the frame; the JSON summary adds the substeps of every frame.  Single GPU only.
// --tap SPEED adds an emitter (SPHSystem's constructor with sphb200::OpenBoundaries, DESIGN.md section 2.6): an 8 x 8 nozzle at the
// fluid spacing, centred above the block at 0.85 of the box height, pointing down, SPEED fast.  --drain SIDE adds a sink on the
// floor: the box [0, SIDE] x [0, 0.05 L] x [0, SIDE] in the (0, 0, 0) corner of the clamp box.  --capacity N is the fluid set's
// capacity (default: twice the initial count).  Single GPU only; they combine with --stir, --float, --vorticity and
// --implicit-viscosity.  The JSON summary then reports fluid_count, emitted, removed and refused.
// --vorticity EPS turns on vorticity confinement of strength EPS (BasicSPHSolver::setVorticityConfinement) after the
// constructor's step 0, for every solver and with --ranks.
// --implicit-viscosity NU turns on the implicit viscosity solve (BasicSPHSolver::setImplicitViscosity) with nu = nu_boundary = NU
// after the constructor's step 0, for every solver: walls and a --stir paddle drag the fluid (no-slip).  Single GPU only, and not
// together with --float (the viscous wall force is not part of a dynamic body's reaction).
// --stir OMEGA adds one kinematic body (SPHSystem's constructor with a KinematicBody): a flat vertical paddle through the
// centre of the fluid block, rotating about y at OMEGA rad/s.  It is two layers of the boundary lattice's spacing thick
// (normal along z), 60 % of the block's x extent wide and as tall as the block; fluid lattice points within one spacing of
// it are dropped.  Single GPU only.
// --float REL adds one dynamic body instead (a KinematicBody with mass > 0, two-way coupled): a hollow cube of side about
// 0.1, its faces sampled at the boundary lattice's spacing, at the centre of the fluid block, initially at rest.  Its mass
// is REL * m0 / spacing^3 * V with V = (extent + boundary spacing)^3, the volume its particles stand for (the fluid's mass
// per unit volume is m0 / spacing^3, DESIGN.md section 2.4), and its moments those of a solid cube of that mass and side.  Fluid lattice points within one spacing of it are dropped.  Single GPU
// only, and not together with --stir.
// --emit-scene writes the generated scene (PREFIX.fluid.f32, PREFIX.boundary.f32; with --tap PREFIX.emitter.f32 = {origin,
// direction, speed, spacing, width, height}; with --drain PREFIX.sink.f32 = {lo, hi}; with --stir also PREFIX.body.f32, the
// paddle's points in body coordinates, and PREFIX.body_state.f32 = pose {c, q = (x, y, z, w)} + motion {V, Omega}; with
// --float the same for the cube and PREFIX.body_dyn.f32 = {M, Ix, Iy, Iz}) and
// exits: needs no GPU, lets a test compare this generator with the python one the benchmarks use, or rebuild the scene.
// --ranks N runs the same scene on N GPUs through SlabSPHSystem (host/sph_slab.hpp: the class API sharded by x-slabs):
// without --rank the process forks one child per GPU (rank r on device r) and a fresh rendezvous directory; with
// --rank R --rendezvous DIR it IS rank R (an external launcher's job).  Every rank dumps the particles it owns
// (PREFIX.rank<R>.*) and prints its own summary line.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <exception>
#include <memory>
#include <string>
#include <vector>

#include <sys/prctl.h>
#include <sys/wait.h>
#include <csignal>
#include <unistd.h>

#include <cuda_runtime.h>

#include "BaseSolver.h"
#include "BasicSPHSolver.h"
#include "DArray.h"
#include "DFSPHSolver.h"
#include "PBDSolver.h"
#include "Particles.h"
#include "SPHParticles.h"
#include "SPHSystem.h"
#include "SlabSPHSystem.h"

namespace {

struct Options {
    std::string solver = "dfsph";
    int frames = 100;
    float box[3] = {1.0f, 1.0f, 1.0f};        // spaceSize, main.cpp:54
    int block[3] = {24, 36, 24};              // fluid block in particles (x, y, z), main.cpp:76-78
    float origin[3] = {0.27f, 0.10f, 0.27f};  // main.cpp:79-81
    float dt = -1.0f;                         // < 0: 0.001 for WCSPH, 0.004 otherwise (README.md:7-9)
    int iters = 0;                            // > 0: fixed iteration count (DFSPH thresholds -1, Q11)
    std::string dump, emitScene;
    bool quiet = false;
    float vorticity = 0.0f;                   // --vorticity EPS: vorticity confinement from frame 1 on (0: off)
    float implicitNu = 0.0f;                  // --implicit-viscosity NU: implicit viscosity from frame 1 on (0: off)
    bool stir = false;                        // --stir OMEGA: a paddle rotating about y at OMEGA rad/s
    float stirOmega = 0.0f;
    bool floating = false;                    // --float REL: a free cube of relative density REL
    float floatRel = 0.0f;
    float tap = 0.0f;                         // --tap SPEED: an emitter above the block (0: none)
    float drain = 0.0f;                       // --drain SIDE: a floor sink (0: none)
    long long capacity = 0;                   // --capacity N: fluid capacity of an open system (0: twice the initial count)
    std::string rheology;                     // --rheology MODEL:PARAMS (empty: off)
    float rheologyMax = -1.0f;                // --rheology-max NU_MAX (< 0: the model's default)
    bool noSlip = false;                      // --no-slip: boundary factor 1 for --rheology
    std::string heat;                         // --heat ALPHA,BETA[,TREF] (empty: off)
    std::string adhesion;                     // --adhesion BETA[,BODYBETA] (empty: off)
    std::string heater, wallTemp, tapTemp, thermalVisc;   // --heater T, --wall-temp T[,H], --tap-temp T, --thermal-viscosity NUREF,E[,NUMAX]
    float cfl = 0.0f;                         // --cfl C: CFL-adaptive substeps, --dt of simulated time per frame (0: off)
    float dtMin = 0.0f;                       // --dt-min X: their smallest dt (0: dt / 64)
    int bullets = 0;                          // test aid: this many top-layer particles start at ~3 cell planes per step
    int ranks = 1, rank = -1;                 // --ranks N: SlabSPHSystem on N GPUs; --rank R: this process is rank R
    std::string rendezvous;
    std::vector<std::string> obstacles;       // --obstacle FILE[,S,X,Y,Z] (repeatable)
    std::string meshBody, fluidMesh;          // --mesh-body FILE,REL[,S,X,Y,Z], --fluid-mesh FILE[,S,X,Y,Z]
    std::vector<std::string> probes, gauges;  // --probe X,Y,Z and --gauge AX,AY,AZ,BX,BY,BZ[,K] (repeatable)
    std::string gaugeThreshold, probeOut;     // --gauge-threshold THETA, --probe-out FILE
    std::string checkpoint, resume;           // --checkpoint FILE, --resume FILE
    int checkpointEvery = 0;                  // --checkpoint-every K (frames; 0: after the last frame only)
    std::string tankRoll, tankShake, tankAccel, tankSpin, tankRamp;   // --tank-* (empty: not given)
    bool tank() const { return !(tankRoll.empty() && tankShake.empty() && tankAccel.empty() && tankSpin.empty() && tankRamp.empty()); }
};

// --rheology MODEL:a,b,c[,d] -> the model (not yet checked against its ranges: setRheology does that)
bool rheology_of(const Options& o, sphb200::Rheology& r) {
    const std::string& spec = o.rheology;
    const size_t colon = spec.find(':');
    if (colon == std::string::npos) return false;
    const std::string model = spec.substr(0, colon);
    std::vector<float> v;
    size_t at = colon + 1;
    while (at <= spec.size()) {
        const size_t comma = std::min(spec.find(',', at), spec.size());
        const std::string item = spec.substr(at, comma - at);
        char* end = nullptr;
        const float x = std::strtof(item.c_str(), &end);
        if (item.empty() || *end != '\0' || !std::isfinite(x)) return false;
        v.push_back(x);
        at = comma + 1;
    }
    const float nuMax = o.rheologyMax;
    if (model == "cross" && v.size() == 4) {
        r = sphb200::Rheology::cross(v[0], v[1], v[2], v[3], nuMax >= 0.0f ? nuMax : std::max(v[0], v[1]));
    } else if (model == "hb" && (v.size() == 3 || v.size() == 4)) {
        r = sphb200::Rheology::herschelBulkley(v[0], v[1], v[2], v.size() == 4 ? v[3] : 1000.0f, nuMax >= 0.0f ? nuMax : 1.0f);
    } else {
        return false;
    }
    return std::isfinite(o.rheologyMax);
}

// "a,b,c" -> finite floats (false for an empty item, a non-number or a non-finite value)
bool floats_of(const std::string& spec, std::vector<float>& v) {
    v.clear();
    size_t at = 0;
    while (at <= spec.size()) {
        const size_t comma = std::min(spec.find(',', at), spec.size());
        const std::string item = spec.substr(at, comma - at);
        char* end = nullptr;
        const float x = std::strtof(item.c_str(), &end);
        if (item.empty() || *end != '\0' || !std::isfinite(x)) return false;
        v.push_back(x);
        at = comma + 1;
    }
    return true;
}

// FILE[,REL][,S,X,Y,Z] of a mesh option
struct MeshSpec {
    std::string file;
    float rel = 0.0f, scale = 1.0f;
    float3 t = {0.0f, 0.0f, 0.0f};
};

bool mesh_spec_of(const std::string& spec, bool withRel, MeshSpec& m) {
    const size_t comma = spec.find(',');
    m = MeshSpec();
    m.file = spec.substr(0, comma);
    std::vector<float> v;
    if (m.file.empty() || (comma != std::string::npos && !floats_of(spec.substr(comma + 1), v))) return false;
    if (withRel) {
        if (v.empty() || !(v[0] >= 0.0f)) return false;
        m.rel = v[0];
        v.erase(v.begin());
    }
    if (!v.empty() && v.size() != 4) return false;
    if (v.size() == 4) { m.scale = v[0]; m.t = make_float3(v[1], v[2], v[3]); }
    return true;
}

// reads and checks one mesh option's mesh before any CUDA call: parsed, closed where required, inside [0, 0.99 box]
bool load_mesh(const char* option, const std::string& spec, bool withRel, bool needClosed, const float box[3], MeshSpec& s,
               sphb200::TriangleMesh& m) {
    if (!mesh_spec_of(spec, withRel, s)) {
        std::fprintf(stderr, "sph_headless: %s needs FILE%s[,S,X,Y,Z] with finite values\n", option, withRel ? ",REL" : "");
        return false;
    }
    try {
        m = sphb200::loadObj(s.file, s.scale, s.t);
        if (needClosed && !sphb200::meshProperties(m).closed) {
            std::fprintf(stderr, "sph_headless: %s %s: the mesh is not closed\n", option, s.file.c_str());
            return false;
        }
    } catch (const std::exception& e) {
        std::fprintf(stderr, "sph_headless: %s %s\n", option, e.what());
        return false;
    }
    for (const float3& v : m.vertices)
        if (!(v.x >= 0.0f && v.y >= 0.0f && v.z >= 0.0f && v.x <= 0.99f * box[0] && v.y <= 0.99f * box[1] && v.z <= 0.99f * box[2])) {
            std::fprintf(stderr, "sph_headless: %s %s: the mesh leaves the box [0, 0.99 * box]\n", option, s.file.c_str());
            return false;
        }
    return true;
}

// --adhesion BETA[,BODYBETA] -> the setting (the walls, and the scene's body if it has one); false for malformed or negative values
bool adhesion_of(const Options& o, bool hasBody, sphb200::Adhesion& a) {
    std::vector<float> v;
    if (!floats_of(o.adhesion, v) || v.size() > 2 || v[0] < 0.0f || v.back() < 0.0f) return false;
    a = sphb200::Adhesion();
    a.wall = v[0];
    if (hasBody) a.bodies.push_back(v.back());
    return true;
}

// --tank-* -> the motion in a box of size `box`; false for malformed values (the ranges are checked by setTankMotion)
bool tank_of(const Options& o, const float box[3], sphb200::TankMotion& m) {
    constexpr double kPi = 3.14159265358979323846;
    m = sphb200::TankMotion();
    m.pivot = make_float3(0.5f * box[0], 0.0f, 0.5f * box[2]);
    m.axis = make_float3(0.0f, o.tankRoll.empty() ? 1.0f : 0.0f, o.tankRoll.empty() ? 0.0f : 1.0f);
    std::vector<float> v;
    if (!o.tankRoll.empty()) {
        if (!floats_of(o.tankRoll, v) || (v.size() != 2 && v.size() != 8) || v[1] < 0.0f) return false;
        m.rollAmplitude = static_cast<float>(v[0] * kPi / 180.0);
        m.rollOmega = static_cast<float>(2.0 * kPi * v[1]);
        if (v.size() == 8) { m.pivot = make_float3(v[2], v[3], v[4]); m.axis = make_float3(v[5], v[6], v[7]); }
    }
    if (!o.tankShake.empty()) {
        if (!floats_of(o.tankShake, v) || v.size() != 4 || v[3] < 0.0f) return false;
        sphb200::TankHarmonic h;
        h.amplitude = make_float3(v[0], v[1], v[2]);
        h.omega = static_cast<float>(2.0 * kPi * v[3]);
        m.harmonics.push_back(h);
    }
    if (!o.tankAccel.empty()) {
        if (!floats_of(o.tankAccel, v) || v.size() != 3) return false;
        m.accel = make_float3(v[0], v[1], v[2]);
    }
    if (!o.tankSpin.empty()) {
        if (!floats_of(o.tankSpin, v) || v.size() != 1) return false;
        m.spin = v[0];
    }
    if (!o.tankRamp.empty()) {
        if (!floats_of(o.tankRamp, v) || v.size() != 1 || v[0] < 0.0f) return false;
        m.ramp = v[0];
    }
    return true;
}

// --probe, --gauge and --gauge-threshold -> the setting (capacity: the caller's); false for malformed or out-of-range values
bool probes_of(const Options& o, sphb200::Probes& p) {
    p = sphb200::Probes();
    for (const auto& spec : o.probes) {
        std::vector<float> v;
        if (!floats_of(spec, v) || v.size() != 3) return false;
        for (float x : v) if (!std::isfinite(x)) return false;
        p.points.push_back(make_float3(v[0], v[1], v[2]));
    }
    for (const auto& spec : o.gauges) {
        std::vector<float> v;
        if (!floats_of(spec, v) || (v.size() != 6 && v.size() != 7)) return false;
        for (float x : v) if (!std::isfinite(x)) return false;
        sphb200::Gauge g;
        g.a = make_float3(v[0], v[1], v[2]);
        g.b = make_float3(v[3], v[4], v[5]);
        if (v.size() == 7) {
            if (v[6] != std::floor(v[6]) || v[6] < 2.0f || v[6] > SPHK_GAUGE_MAX_SAMPLES) return false;
            g.samples = static_cast<int>(v[6]);
        }
        if (g.a.x == g.b.x && g.a.y == g.b.y && g.a.z == g.b.z) return false;
        p.gauges.push_back(g);
    }
    if (!o.gaugeThreshold.empty()) {
        std::vector<float> v;
        if (!floats_of(o.gaugeThreshold, v) || v.size() != 1 || !std::isfinite(v[0]) || !(v[0] > 0.0f)) return false;
        p.threshold = v[0];
    }
    return p.points.size() <= SPHK_PROBE_LIMIT && p.gauges.size() <= SPHK_GAUGE_LIMIT;
}

// --heat and its companions -> the thermal setting and the viscosity law (ranges are checked by the setters)
bool thermal_of(const Options& o, sphb200::Thermal& t, sphb200::ThermalViscosity& tv) {
    std::vector<float> v;
    if (!floats_of(o.heat, v) || v.size() < 2 || v.size() > 3) return false;
    t = sphb200::Thermal();
    t.alpha = v[0]; t.beta = v[1]; t.Tref = v.size() == 3 ? v[2] : 0.0f;
    t.wall = {t.Tref, 0.0f};
    if (!o.wallTemp.empty()) {
        if (!floats_of(o.wallTemp, v) || v.size() > 2) return false;
        t.wall = {v[0], v.size() == 2 ? v[1] : 1.0f};
    }
    if (!o.heater.empty()) {
        if (!floats_of(o.heater, v) || v.size() != 1) return false;
        t.bodies.push_back({v[0], 1.0f});
    }
    if (!o.tapTemp.empty()) {
        if (!floats_of(o.tapTemp, v) || v.size() != 1) return false;
        t.emitterT.push_back(v[0]);
    }
    if (!o.thermalVisc.empty()) {
        if (!floats_of(o.thermalVisc, v) || v.size() < 2 || v.size() > 3) return false;
        tv = sphb200::ThermalViscosity();
        tv.nuRef = v[0]; tv.E = v[1]; tv.nuMax = v.size() == 3 ? v[2] : 100.0f * v[0]; tv.wallFactor = 1.0f;
    }
    return true;
}

bool parse(int argc, char** argv, Options& o) {
    auto need = [&](int i, int k) { return i + k < argc; };
    for (int i = 1; i < argc; ++i) {
        const std::string a = argv[i];
        if (a == "--solver" && need(i, 1)) o.solver = argv[++i];
        else if (a == "--frames" && need(i, 1)) o.frames = std::atoi(argv[++i]);
        else if (a == "--dt" && need(i, 1)) o.dt = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--iters" && need(i, 1)) o.iters = std::atoi(argv[++i]);
        else if (a == "--dump" && need(i, 1)) o.dump = argv[++i];
        else if (a == "--emit-scene" && need(i, 1)) o.emitScene = argv[++i];
        else if (a == "--quiet") o.quiet = true;
        else if (a == "--bullets" && need(i, 1)) o.bullets = std::atoi(argv[++i]);
        else if (a == "--vorticity" && need(i, 1)) o.vorticity = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--implicit-viscosity" && need(i, 1)) o.implicitNu = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--stir" && need(i, 1)) { o.stir = true; o.stirOmega = static_cast<float>(std::atof(argv[++i])); }
        else if (a == "--float" && need(i, 1)) { o.floating = true; o.floatRel = static_cast<float>(std::atof(argv[++i])); }
        else if (a == "--tap" && need(i, 1)) o.tap = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--drain" && need(i, 1)) o.drain = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--capacity" && need(i, 1)) o.capacity = std::atoll(argv[++i]);
        else if (a == "--rheology" && need(i, 1)) o.rheology = argv[++i];
        else if (a == "--rheology-max" && need(i, 1)) o.rheologyMax = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--no-slip") o.noSlip = true;
        else if (a == "--heat" && need(i, 1)) o.heat = argv[++i];
        else if (a == "--adhesion" && need(i, 1)) o.adhesion = argv[++i];
        else if (a == "--tank-roll" && need(i, 1)) o.tankRoll = argv[++i];
        else if (a == "--tank-shake" && need(i, 1)) o.tankShake = argv[++i];
        else if (a == "--tank-accel" && need(i, 1)) o.tankAccel = argv[++i];
        else if (a == "--tank-spin" && need(i, 1)) o.tankSpin = argv[++i];
        else if (a == "--tank-ramp" && need(i, 1)) o.tankRamp = argv[++i];
        else if (a == "--heater" && need(i, 1)) o.heater = argv[++i];
        else if (a == "--wall-temp" && need(i, 1)) o.wallTemp = argv[++i];
        else if (a == "--tap-temp" && need(i, 1)) o.tapTemp = argv[++i];
        else if (a == "--thermal-viscosity" && need(i, 1)) o.thermalVisc = argv[++i];
        else if (a == "--cfl" && need(i, 1)) o.cfl = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--dt-min" && need(i, 1)) o.dtMin = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--ranks" && need(i, 1)) o.ranks = std::atoi(argv[++i]);
        else if (a == "--rank" && need(i, 1)) o.rank = std::atoi(argv[++i]);
        else if (a == "--rendezvous" && need(i, 1)) o.rendezvous = argv[++i];
        else if (a == "--obstacle" && need(i, 1)) o.obstacles.push_back(argv[++i]);
        else if (a == "--mesh-body" && need(i, 1)) o.meshBody = argv[++i];
        else if (a == "--fluid-mesh" && need(i, 1)) o.fluidMesh = argv[++i];
        else if (a == "--probe" && need(i, 1)) o.probes.push_back(argv[++i]);
        else if (a == "--gauge" && need(i, 1)) o.gauges.push_back(argv[++i]);
        else if (a == "--gauge-threshold" && need(i, 1)) o.gaugeThreshold = argv[++i];
        else if (a == "--probe-out" && need(i, 1)) o.probeOut = argv[++i];
        else if (a == "--checkpoint" && need(i, 1)) o.checkpoint = argv[++i];
        else if (a == "--resume" && need(i, 1)) o.resume = argv[++i];
        else if (a == "--checkpoint-every" && need(i, 1)) {
            char* end = nullptr;
            const long k = std::strtol(argv[++i], &end, 10);
            o.checkpointEvery = (end && *end == 0 && k >= 0 && k <= 1000000000L) ? static_cast<int>(k) : -1;
        }
        else if (a == "--block" && need(i, 3)) { for (int k = 0; k < 3; ++k) o.block[k] = std::atoi(argv[++i]); }
        else if (a == "--origin" && need(i, 3)) { for (int k = 0; k < 3; ++k) o.origin[k] = static_cast<float>(std::atof(argv[++i])); }
        else if (a == "--box" && need(i, 1)) {
            o.box[0] = static_cast<float>(std::atof(argv[++i]));
            if (need(i, 2) && argv[i + 1][0] != '-' && argv[i + 2][0] != '-') {
                o.box[1] = static_cast<float>(std::atof(argv[++i]));
                o.box[2] = static_cast<float>(std::atof(argv[++i]));
            } else {
                o.box[1] = o.box[2] = o.box[0];
            }
        } else {
            std::fprintf(stderr, "sph_headless: unknown or incomplete option '%s'\n", a.c_str());
            return false;
        }
    }
    if (o.ranks < 1 || o.rank >= o.ranks || (o.rank >= 0 && o.ranks > 1 && o.rendezvous.empty())) return false;
    if (o.stir && (o.ranks > 1 || !std::isfinite(o.stirOmega))) {
        std::fprintf(stderr, "sph_headless: --stir runs on one GPU only (kinematic bodies are not supported with --ranks)\n");
        return false;
    }
    if (o.floating && (o.ranks > 1 || o.stir || !(o.floatRel > 0.0f) || !std::isfinite(o.floatRel))) {
        std::fprintf(stderr, "sph_headless: --float REL needs REL > 0, runs on one GPU only (bodies are not supported with --ranks) "
                             "and not together with --stir\n");
        return false;
    }
    if (!(o.implicitNu >= 0.0f) || !std::isfinite(o.implicitNu)) {
        std::fprintf(stderr, "sph_headless: --implicit-viscosity NU needs a finite NU >= 0\n");
        return false;
    }
    if (o.implicitNu > 0.0f && (o.ranks > 1 || o.floating)) {
        std::fprintf(stderr, "sph_headless: --implicit-viscosity runs on one GPU only (not with --ranks) and not together with --float\n");
        return false;
    }
    if (!(o.tap >= 0.0f) || !std::isfinite(o.tap) || !(o.drain >= 0.0f) || !std::isfinite(o.drain) || o.capacity < 0 ||
        o.capacity > 0x7fffffffLL) {
        std::fprintf(stderr, "sph_headless: --tap SPEED and --drain SIDE need finite values > 0, --capacity N a count\n");
        return false;
    }
    if ((o.tap > 0.0f || o.drain > 0.0f) && o.ranks > 1) {
        std::fprintf(stderr, "sph_headless: --tap and --drain run on one GPU only (open boundaries are not supported with --ranks)\n");
        return false;
    }
    if (!o.rheology.empty()) {
        sphb200::Rheology r;
        if (!rheology_of(o, r)) {
            std::fprintf(stderr, "sph_headless: --rheology needs cross:NU0,NUINF,LAMBDA,M or hb:K,N,TAU[,MREG] with finite values\n");
            return false;
        }
        if (o.ranks > 1 || o.implicitNu > 0.0f || (o.noSlip && o.floating)) {
            std::fprintf(stderr, "sph_headless: --rheology runs on one GPU only (not with --ranks), not together with --implicit-viscosity, "
                                 "and --no-slip not together with --float\n");
            return false;
        }
    } else if (o.noSlip || o.rheologyMax >= 0.0f) {
        std::fprintf(stderr, "sph_headless: --no-slip and --rheology-max go with --rheology\n");
        return false;
    }
    if (!o.heat.empty()) {
        sphb200::Thermal t;
        sphb200::ThermalViscosity tv;
        if (!thermal_of(o, t, tv)) {
            std::fprintf(stderr, "sph_headless: --heat needs ALPHA,BETA[,TREF], --heater T, --wall-temp T[,H], --tap-temp T and "
                                 "--thermal-viscosity NUREF,E[,NUMAX] with finite values\n");
            return false;
        }
        if (o.ranks > 1 || (!o.heater.empty() && (o.stir || o.floating)) || (!o.tapTemp.empty() && !(o.tap > 0.0f)) ||
            (!o.thermalVisc.empty() && (!o.rheology.empty() || o.implicitNu > 0.0f || o.floating))) {
            std::fprintf(stderr, "sph_headless: --heat runs on one GPU only (not with --ranks); --heater not together with --stir or "
                                 "--float; --tap-temp needs --tap; --thermal-viscosity not together with --rheology, "
                                 "--implicit-viscosity or --float\n");
            return false;
        }
    } else if (!o.heater.empty() || !o.wallTemp.empty() || !o.tapTemp.empty() || !o.thermalVisc.empty()) {
        std::fprintf(stderr, "sph_headless: --heater, --wall-temp, --tap-temp and --thermal-viscosity go with --heat\n");
        return false;
    }
    if (!o.adhesion.empty()) {
        sphb200::Adhesion a;
        if (!adhesion_of(o, false, a) || o.ranks > 1) {
            std::fprintf(stderr, "sph_headless: --adhesion needs BETA[,BODYBETA] with finite values >= 0 and runs on one GPU only (not "
                                 "with --ranks)\n");
            return false;
        }
    }
    if (!(o.cfl >= 0.0f) || !std::isfinite(o.cfl) || !(o.dtMin >= 0.0f) || !std::isfinite(o.dtMin)) {
        std::fprintf(stderr, "sph_headless: --cfl C and --dt-min X need finite values > 0\n");
        return false;
    }
    if (o.cfl > 0.0f && o.ranks > 1) {
        std::fprintf(stderr, "sph_headless: --cfl runs on one GPU only (adaptive time stepping is not supported with --ranks)\n");
        return false;
    }
    if ((!o.obstacles.empty() || !o.meshBody.empty() || !o.fluidMesh.empty()) && o.ranks > 1) {
        std::fprintf(stderr, "sph_headless: --obstacle, --mesh-body and --fluid-mesh run on one GPU only (not with --ranks)\n");
        return false;
    }
    if (!o.checkpoint.empty() || !o.resume.empty() || o.checkpointEvery != 0) {
        if (o.checkpointEvery < 0 || (o.checkpointEvery > 0 && o.checkpoint.empty()) || o.ranks > 1 || o.bullets > 0 || o.frames < 0) {
            std::fprintf(stderr, "sph_headless: --checkpoint FILE, --checkpoint-every K (an integer >= 0, with --checkpoint) and --resume FILE "
                                 "run on one GPU only (not with --ranks) and not with --bullets\n");
            return false;
        }
    }
    if (!o.probes.empty() || !o.gauges.empty() || !o.gaugeThreshold.empty() || !o.probeOut.empty()) {
        sphb200::Probes p;
        if (!probes_of(o, p) || o.ranks > 1 || o.probeOut.empty() || (p.points.empty() && p.gauges.empty()) ||
            (!o.gaugeThreshold.empty() && p.gauges.empty())) {
            std::fprintf(stderr, "sph_headless: --probe X,Y,Z and --gauge AX,AY,AZ,BX,BY,BZ[,K] need finite values, a != b and K in [2, %d] "
                                 "(at most %d probes and %d gauges), --gauge-threshold a finite value > 0 and gauges, --probe-out a file "
                                 "and at least one probe or gauge; single GPU only (not with --ranks)\n",
                         SPHK_GAUGE_MAX_SAMPLES, SPHK_PROBE_LIMIT, SPHK_GAUGE_LIMIT);
            return false;
        }
    }
    if (o.tank()) {
        sphb200::TankMotion m;
        if (!tank_of(o, o.box, m) || o.ranks > 1 || !o.heat.empty()) {
            std::fprintf(stderr, "sph_headless: --tank-roll DEG,HZ[,PX,PY,PZ,NX,NY,NZ], --tank-shake AX,AY,AZ,HZ, --tank-accel AX,AY,AZ, "
                                 "--tank-spin RAD_S and --tank-ramp SEC need finite values (HZ, SEC >= 0); single GPU only (not with "
                                 "--ranks) and not with --heat\n");
            return false;
        }
    }
    if (!o.meshBody.empty() && (o.stir || o.floating || !o.heater.empty())) {
        std::fprintf(stderr, "sph_headless: --mesh-body not together with --stir, --float or --heater\n");
        return false;
    }
    return o.frames >= 0 && o.vorticity >= 0.0f && o.block[0] > 0 && o.block[1] > 0 && o.block[2] > 0 &&
           (o.solver == "sph" || o.solver == "wcsph" || o.solver == "dfsph" || o.solver == "pbd");
}

// fluid block: y outermost, then x, z innermost (the order fixes the initial particle numbering)
std::vector<float3> fluid_block(const Options& o, float spacing) {
    std::vector<float3> p;
    p.reserve(static_cast<size_t>(o.block[0]) * o.block[1] * o.block[2]);
    for (int iy = 0; iy < o.block[1]; ++iy)
        for (int ix = 0; ix < o.block[0]; ++ix)
            for (int iz = 0; iz < o.block[2]; ++iz)
                p.push_back(make_float3(o.origin[0] + spacing * ix, o.origin[1] + spacing * iy, o.origin[2] + spacing * iz));
    return p;
}

// boundary shell: the six faces of a (2*cells)^3 lattice squeezed by 0.99 into the box; pairs of opposite faces are
// emitted together, front/back first, then bottom/top without the edges already emitted, then left/right
std::vector<float3> boundary_shell(const int3 cells, const float3 space) {
    const int3 c = make_int3(2 * cells.x, 2 * cells.y, 2 * cells.z);
    std::vector<float3> p;
    auto put = [&](int i, int j, int k) {
        const float3 x = make_float3(float(i) / float(c.x - 1) * space.x, float(j) / float(c.y - 1) * space.y,
                                     float(k) / float(c.z - 1) * space.z);
        p.push_back(make_float3(0.99f * x.x + 0.005f * space.x, 0.99f * x.y + 0.005f * space.y, 0.99f * x.z + 0.005f * space.z));
    };
    for (int i = 0; i < c.x; ++i)
        for (int j = 0; j < c.y; ++j) { put(i, j, 0); put(i, j, c.z - 1); }
    for (int i = 0; i < c.x; ++i)
        for (int k = 0; k < c.z - 2; ++k) { put(i, 0, k + 1); put(i, c.y - 1, k + 1); }
    for (int j = 0; j < c.y - 2; ++j)
        for (int k = 0; k < c.z - 2; ++k) { put(0, j + 1, k + 1); put(c.x - 1, j + 1, k + 1); }
    return p;
}

// --stir: the paddle (body coordinates, centred on the block's centre) and the fluid block without the lattice points
// within one boundary spacing of it
sphb200::KinematicBody paddle(const Options& o, float spacing, float boundarySpacing) {
    sphb200::KinematicBody b;
    const float sb = boundarySpacing;
    const float ex = spacing * (o.block[0] - 1), ey = spacing * (o.block[1] - 1);
    const int nw = std::max(2, static_cast<int>(0.6f * ex / sb) + 1), nh = std::max(2, static_cast<int>(ey / sb) + 1);
    for (int j = 0; j < nh; ++j)
        for (int i = 0; i < nw; ++i)
            for (int k = 0; k < 2; ++k)
                b.points.push_back(make_float3((i - 0.5f * (nw - 1)) * sb, (j - 0.5f * (nh - 1)) * sb, (k - 0.5f) * sb));
    b.position = make_float3(o.origin[0] + 0.5f * ex, o.origin[1] + 0.5f * ey, o.origin[2] + 0.5f * spacing * (o.block[2] - 1));
    b.orientation = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
    b.linearVelocity = make_float3(0.0f, 0.0f, 0.0f);
    b.angularVelocity = make_float3(0.0f, o.stirOmega, 0.0f);
    return b;
}

constexpr float kSphM0 = 76.596750762082e-6f;   // the fluid particle mass m0, main.cpp

// --heater: a held plate (two boundary layers) on the floor under the block, one spacing wider than the block on every side
sphb200::KinematicBody heater_plate(const Options& o, float spacing, float boundarySpacing) {
    sphb200::KinematicBody b;
    const float sb = boundarySpacing;
    const float ex = spacing * (o.block[0] - 1) + 2.0f * spacing, ez = spacing * (o.block[2] - 1) + 2.0f * spacing;
    const int nx = std::max(2, static_cast<int>(ex / sb) + 1), nz = std::max(2, static_cast<int>(ez / sb) + 1);
    for (int i = 0; i < nx; ++i)
        for (int k = 0; k < nz; ++k)
            for (int j = 0; j < 2; ++j)
                b.points.push_back(make_float3((i - 0.5f * (nx - 1)) * sb, (j - 0.5f) * sb, (k - 0.5f * (nz - 1)) * sb));
    b.position = make_float3(o.origin[0] + 0.5f * spacing * (o.block[0] - 1), 2.5f * sb,
                             o.origin[2] + 0.5f * spacing * (o.block[2] - 1));
    b.orientation = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
    b.linearVelocity = make_float3(0.0f, 0.0f, 0.0f);
    b.angularVelocity = make_float3(0.0f, 0.0f, 0.0f);
    return b;
}

// --float: the hollow cube (body coordinates, centred on the block's centre, at rest), mass and moments of a solid cube
sphb200::KinematicBody floating_cube(const Options& o, float spacing, float boundarySpacing) {
    sphb200::KinematicBody b;
    const float sb = boundarySpacing;
    const int n = std::max(2, static_cast<int>(std::lround(0.1f / sb)) + 1);
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j)
            for (int k = 0; k < n; ++k)
                if (i == 0 || j == 0 || k == 0 || i == n - 1 || j == n - 1 || k == n - 1)
                    b.points.push_back(make_float3((i - 0.5f * (n - 1)) * sb, (j - 0.5f * (n - 1)) * sb, (k - 0.5f * (n - 1)) * sb));
    const float ex = spacing * (o.block[0] - 1), ey = spacing * (o.block[1] - 1);
    b.position = make_float3(o.origin[0] + 0.5f * ex, o.origin[1] + 0.5f * ey, o.origin[2] + 0.5f * spacing * (o.block[2] - 1));
    b.orientation = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
    b.linearVelocity = make_float3(0.0f, 0.0f, 0.0f);
    b.angularVelocity = make_float3(0.0f, 0.0f, 0.0f);
    const float side = n * sb;           // the volume its particles stand for: (extent + spacing)^3
    b.mass = o.floatRel * (kSphM0 / (spacing * spacing * spacing)) * side * side * side;
    const float I = b.mass * side * side / 6.0f;
    b.inertia = make_float3(I, I, I);
    return b;
}

std::vector<float3> clear_of(const std::vector<float3>& fluid, const sphb200::KinematicBody& b, float sb) {
    float3 lo = b.points[0], hi = b.points[0];
    for (const float3& r : b.points) {
        lo = make_float3(std::min(lo.x, r.x), std::min(lo.y, r.y), std::min(lo.z, r.z));
        hi = make_float3(std::max(hi.x, r.x), std::max(hi.y, r.y), std::max(hi.z, r.z));
    }
    std::vector<float3> out;
    for (const float3& p : fluid) {
        const float dx = p.x - b.position.x, dy = p.y - b.position.y, dz = p.z - b.position.z;   // identity orientation at t = 0
        const float ox = std::max({lo.x - dx, dx - hi.x, 0.0f}), oy = std::max({lo.y - dy, dy - hi.y, 0.0f}),
                    oz = std::max({lo.z - dz, dz - hi.z, 0.0f});
        if (ox * ox + oy * oy + oz * oz >= sb * sb) out.push_back(p);
    }
    return out;
}

// --tap / --drain (DESIGN.md section 2.6)
sphb200::OpenBoundaries open_boundaries(const Options& o, float spacing) {
    sphb200::OpenBoundaries ob;
    if (o.tap > 0.0f) {
        sphb200::Emitter e;
        e.origin = make_float3(o.origin[0] + 0.5f * spacing * (o.block[0] - 1), 0.85f * o.box[1], o.origin[2] + 0.5f * spacing * (o.block[2] - 1));
        e.direction = make_float3(0.0f, -1.0f, 0.0f);
        e.speed = o.tap;
        e.spacing = spacing;
        e.width = e.height = 8;
        ob.emitters.push_back(e);
    }
    if (o.drain > 0.0f) ob.sinks.push_back({make_float3(0.0f, 0.0f, 0.0f), make_float3(o.drain, 0.05f * o.box[1], o.drain)});
    return ob;
}

std::vector<float> flat(const std::vector<float3>& p) {
    std::vector<float> v;
    v.reserve(3 * p.size());
    for (const float3& q : p) { v.push_back(q.x); v.push_back(q.y); v.push_back(q.z); }
    return v;
}

bool write_floats(const std::string& path, const std::vector<float>& v) {
    FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) return false;
    const bool ok = std::fwrite(v.data(), sizeof(float), v.size(), f) == v.size();
    std::fclose(f);
    return ok;
}

// --bullets: the chosen top-layer lattice particles (found by position among slots [begin, begin + count): the lattice
// survives the constructor's step 0) get a velocity of about three cell planes per step, alternately +x / -x, and upwards.
// What a violent impact does to a few particles; on several GPUs it exercises the stray routing of SlabSPHSystem.
int shoot(const Options& o, float spacing, float dt, const std::shared_ptr<SPHParticles>& fluids, size_t begin, size_t count) {
    if (o.bullets <= 0 || count == 0) return 0;
    std::vector<float3> pos(count), vel(count);
    if (cudaMemcpy(pos.data(), fluids->getPosPtr() + begin, count * sizeof(float3), cudaMemcpyDeviceToHost) != cudaSuccess ||
        cudaMemcpy(vel.data(), fluids->getVelPtr() + begin, count * sizeof(float3), cudaMemcpyDeviceToHost) != cudaSuccess)
        return -1;
    const float speed = 30.0f * 0.004f / dt;
    int hit = 0;
    for (size_t i = 0; i < count; ++i) {
        const int ix = static_cast<int>(std::lround((pos[i].x - o.origin[0]) / spacing)), iy = static_cast<int>(std::lround((pos[i].y - o.origin[1]) / spacing)),
                  iz = static_cast<int>(std::lround((pos[i].z - o.origin[2]) / spacing));
        if (iy != o.block[1] - 1) continue;
        for (int b = 0; b < o.bullets; ++b)
            if (ix == static_cast<int>((b + 0.5) * o.block[0] / o.bullets) && iz == o.block[2] / 2 + (b % 3) - 1) {
                const float3 v = make_float3(b % 2 == 0 ? speed : -speed, 0.7f * speed, 0.0f);
                if (o.solver == "pbd")      // PBD derives the velocity from the positions (PBDSolver.cu:56): displace the particle instead
                    pos[i] = make_float3(pos[i].x + dt * v.x, pos[i].y + dt * v.y, pos[i].z + dt * v.z);
                else
                    vel[i] = v;
                ++hit;
            }
    }
    if (hit && (cudaMemcpy(fluids->getVelPtr() + begin, vel.data(), count * sizeof(float3), cudaMemcpyHostToDevice) != cudaSuccess ||
                cudaMemcpy(fluids->getPosPtr() + begin, pos.data(), count * sizeof(float3), cudaMemcpyHostToDevice) != cudaSuccess))
        return -1;
    return hit;
}

}  // namespace

int main(int argc, char** argv) {
    Options o;
    if (!parse(argc, argv, o)) {
        std::fprintf(stderr, "usage: sph_headless [--solver sph|dfsph|pbd] [--frames N] [--box L | LX LY LZ] [--block NX NY NZ] "
                             "[--origin X Y Z] [--dt DT] [--iters K] [--vorticity EPS] [--implicit-viscosity NU] [--stir OMEGA | --float REL] "
                             "[--tap SPEED] [--drain SIDE] [--capacity N] [--cfl C [--dt-min X]] [--rheology cross:NU0,NUINF,LAMBDA,M | hb:K,N,TAU[,MREG] "
                             "[--rheology-max NU_MAX] [--no-slip]] [--heat ALPHA,BETA[,TREF] [--heater T] [--wall-temp T[,H]] "
                             "[--tap-temp T] [--thermal-viscosity NUREF,E[,NUMAX]]] [--adhesion BETA[,BODYBETA]] [--obstacle FILE[,S,X,Y,Z]]... "
                             "[--mesh-body FILE,REL[,S,X,Y,Z]] [--fluid-mesh FILE[,S,X,Y,Z]] [--dump PREFIX] [--quiet] "
                             "[--tank-roll DEG,HZ[,PX,PY,PZ,NX,NY,NZ]] [--tank-shake AX,AY,AZ,HZ] [--tank-accel AX,AY,AZ] [--tank-spin RAD_S] "
                             "[--tank-ramp SEC] "
                             "[--emit-scene PREFIX] [--checkpoint FILE [--checkpoint-every K]] [--resume FILE] "
                             "[--ranks N [--rank R --rendezvous DIR]]\n");
        return 2;
    }
    // ---- scene constants, main.cpp:54-67 ----
    const float3 spaceSize = make_float3(o.box[0], o.box[1], o.box[2]);
    const float sphSpacing = 0.02f;
    const float sphSmoothingRadius = 2.0f * sphSpacing;
    const float sphCellLength = 1.01f * sphSmoothingRadius;
    const int3 cellSize = make_int3(static_cast<int>(std::ceil(spaceSize.x / sphCellLength)), static_cast<int>(std::ceil(spaceSize.y / sphCellLength)),
                                    static_cast<int>(std::ceil(spaceSize.z / sphCellLength)));
    // the boundary shell's lattice spacing along x (boundary_shell: 0.99 * space / (2 * cells - 1))
    const float boundarySpacing = 0.99f * spaceSize.x / float(2 * cellSize.x - 1);
    // ---- meshes: read and checked before any CUDA call ----
    std::vector<sphb200::TriangleMesh> carve;               // the obstacles, then the body: the fluid is cleared of them
    sphb200::TriangleMesh bodyMesh, fluidMesh;
    MeshSpec spec;
    for (const std::string& ob : o.obstacles) {
        carve.emplace_back();
        if (!load_mesh("--obstacle", ob, false, true, o.box, spec, carve.back())) return 2;
    }
    const size_t nObstacles = carve.size();
    float meshRel = 0.0f;
    if (!o.meshBody.empty()) {
        if (!load_mesh("--mesh-body", o.meshBody, true, true, o.box, spec, bodyMesh)) return 2;
        meshRel = spec.rel;
        carve.push_back(bodyMesh);
    }
    if (!o.fluidMesh.empty() && !load_mesh("--fluid-mesh", o.fluidMesh, false, true, o.box, spec, fluidMesh)) return 2;
    std::vector<sphb200::KinematicBody> bodies;
    std::vector<float3> fluidPoints, boundaryPoints = boundary_shell(cellSize, spaceSize);
    try {
        fluidPoints = o.fluidMesh.empty() ? fluid_block(o, sphSpacing)
                                          : sphb200::fillMesh(fluidMesh, sphSpacing, make_float3(o.origin[0], o.origin[1], o.origin[2]), 0.0f);
        for (size_t k = 0; k < nObstacles; ++k) {
            const std::vector<float3> s = sphb200::sampleSurface(carve[k], boundarySpacing);
            boundaryPoints.insert(boundaryPoints.end(), s.begin(), s.end());
        }
        if (!o.meshBody.empty())
            bodies.push_back(sphb200::meshBody(bodyMesh, boundarySpacing, meshRel, kSphM0 / (sphSpacing * sphSpacing * sphSpacing)));
        if (!carve.empty()) fluidPoints = sphb200::clearOf(fluidPoints, carve, boundarySpacing);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "sph_headless: building the mesh scene failed: %s\n", e.what());
        return 4;
    }
    if (o.stir) bodies.push_back(paddle(o, sphSpacing, boundarySpacing));
    if (o.floating) bodies.push_back(floating_cube(o, sphSpacing, boundarySpacing));
    if (!o.heater.empty()) bodies.push_back(heater_plate(o, sphSpacing, boundarySpacing));
    if (!bodies.empty() && o.meshBody.empty()) fluidPoints = clear_of(fluidPoints, bodies[0], boundarySpacing);
    const sphb200::OpenBoundaries openB = open_boundaries(o, sphSpacing);
    const bool open = !openB.emitters.empty() || !openB.sinks.empty();
    if (!o.emitScene.empty()) {
        const int3 cells = cellSize;
        bool ok = write_floats(o.emitScene + ".fluid.f32", flat(fluidPoints)) &&
                  write_floats(o.emitScene + ".boundary.f32", flat(boundaryPoints));
        if (ok && !bodies.empty()) {
            const auto& b = bodies[0];
            ok = write_floats(o.emitScene + ".body.f32", flat(b.points)) &&
                 write_floats(o.emitScene + ".body_state.f32",
                              {b.position.x, b.position.y, b.position.z, b.orientation.x, b.orientation.y, b.orientation.z, b.orientation.w,
                               b.linearVelocity.x, b.linearVelocity.y, b.linearVelocity.z, b.angularVelocity.x, b.angularVelocity.y,
                               b.angularVelocity.z});
            if (ok && (o.floating || !o.meshBody.empty()))
                ok = write_floats(o.emitScene + ".body_dyn.f32", {b.mass, b.inertia.x, b.inertia.y, b.inertia.z});
        }
        for (const auto& e : openB.emitters)
            ok = ok && write_floats(o.emitScene + ".emitter.f32", {e.origin.x, e.origin.y, e.origin.z, e.direction.x, e.direction.y, e.direction.z,
                                                                    e.speed, e.spacing, float(e.width), float(e.height)});
        for (const auto& b : openB.sinks)
            ok = ok && write_floats(o.emitScene + ".sink.f32", {b.lo.x, b.lo.y, b.lo.z, b.hi.x, b.hi.y, b.hi.z});
        std::printf("{\"cells\": [%d, %d, %d]}\n", cells.x, cells.y, cells.z);
        return ok ? 0 : 5;
    }
    // ---- --ranks N without --rank: one child per GPU, forked BEFORE the first CUDA call of this process ----
    if (o.ranks > 1 && o.rank < 0) {
        char tmpl[] = "/tmp/sph_headless_rdv_XXXXXX";
        if (!mkdtemp(tmpl)) { std::perror("sph_headless: mkdtemp"); return 5; }
        o.rendezvous = tmpl;
        std::vector<pid_t> kids;
        for (int r = 0; r < o.ranks; ++r) {
            std::fflush(nullptr);
            const pid_t pid = fork();
            if (pid < 0) { std::perror("sph_headless: fork"); return 5; }
            if (pid == 0) { prctl(PR_SET_PDEATHSIG, SIGKILL); o.rank = r; kids.clear(); break; }   // never outlive the launcher
            kids.push_back(pid);
        }
        if (o.rank < 0) {
            int worstRc = 0;
            for (size_t left = kids.size(); left > 0; --left) {
                int st = 0;
                const pid_t done = waitpid(-1, &st, 0);
                if (done < 0) break;
                const int rc = WIFEXITED(st) ? WEXITSTATUS(st) : 128;
                if (rc != 0 && worstRc == 0) {          // a rank that failed cannot be waited for by the others: end the job
                    worstRc = rc;                       // (and report ITS exit code, not that of the ranks killed here)
                    for (const pid_t pid : kids)
                        if (pid != done) kill(pid, SIGKILL);
                }
            }
            for (const char* f : {"nccl_id"}) std::remove((o.rendezvous + "/" + f).c_str());
            for (int r = 0; r < o.ranks; ++r)
                for (const char* f : {"ipc_", "connected_"}) std::remove((o.rendezvous + "/" + f + std::to_string(r)).c_str());
            rmdir(o.rendezvous.c_str());
            return worstRc;
        }
    }
    const bool slab = o.ranks > 1;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        std::fprintf(stderr, "sph_headless: no CUDA device -- this engine has no CPU path\n");
        return 3;
    }
    if (slab) {
        if (ndev < o.ranks) { std::fprintf(stderr, "sph_headless: --ranks %d needs %d GPUs, this box has %d\n", o.ranks, o.ranks, ndev); return 3; }
        if (cudaSetDevice(o.rank) != cudaSuccess) { std::fprintf(stderr, "sph_headless: cudaSetDevice(%d) failed\n", o.rank); return 3; }
        o.quiet = o.quiet || o.rank != 0;
    }
    const bool wcsph = (o.solver == "sph" || o.solver == "wcsph");
    const float dt = o.dt > 0.0f ? o.dt : (wcsph ? 0.001f : 0.004f);
    const float sphRho0 = 1.0f;
    const float sphRhoBoundary = 1.4f * sphRho0;
    const float sphM0 = kSphM0;
    const float sphStiff = 10.0f;
    const float3 sphG = make_float3(0.0f, -9.8f, 0.0f);
    const float sphVisc = 5e-4f;
    const float sphSurfaceTensionIntensity = 0.0001f;
    const float sphAirPressure = 0.0001f;

    // ---- the reference's call sites: particles (main.cpp:86,117), solver (:119-130), system (:131-134) ----
    const unsigned int capacity = open ? static_cast<unsigned int>(o.capacity > 0 ? o.capacity : 2LL * static_cast<long long>(fluidPoints.size()))
                                       : static_cast<unsigned int>(fluidPoints.size());
    auto fluidParticles = open ? std::make_shared<SPHParticles>(fluidPoints, capacity) : std::make_shared<SPHParticles>(fluidPoints);
    auto boundaryParticles = std::make_shared<SPHParticles>(boundaryPoints);
    const int nFluid = static_cast<int>(fluidParticles->size()), nBoundary = static_cast<int>(boundaryParticles->size());
    const int nSlots = static_cast<int>(fluidParticles->capacity());   // the solver's buffers hold every slot
    std::shared_ptr<BaseSolver> pSolver;
    if (o.solver == "pbd")
        pSolver = o.iters > 0 ? std::make_shared<PBDSolver>(nSlots, o.iters) : std::make_shared<PBDSolver>(nSlots);
    else if (o.solver == "dfsph")
        pSolver = o.iters > 0 ? std::make_shared<DFSPHSolver>(nSlots, -1.0f, -1.0f, o.iters) : std::make_shared<DFSPHSolver>(nSlots);
    else
        pSolver = std::make_shared<BasicSPHSolver>(nSlots);
    BasicSPHSolver* basicSolver = dynamic_cast<BasicSPHSolver*>(pSolver.get());   // (the systems take pSolver over)
    std::shared_ptr<SPHSystem> pSystem;
    std::shared_ptr<SlabSPHSystem> pSlab;
    if (slab) {
        sphb200::SlabBootstrap boot;
        boot.rank = o.rank; boot.world = o.ranks; boot.rendezvousDir = o.rendezvous;
        pSlab = std::make_shared<SlabSPHSystem>(fluidParticles, boundaryParticles, pSolver, spaceSize, sphCellLength, sphSmoothingRadius,
                                                dt, sphM0, sphRho0, sphRhoBoundary, sphStiff, sphVisc, sphSurfaceTensionIntensity,
                                                sphAirPressure, sphG, cellSize, boot);
        if (!pSlab->ok()) { std::fprintf(stderr, "sph_headless: rank %d: SlabSPHSystem did not come up\n", o.rank); return 4; }
    } else if (open) {
        pSystem = std::make_shared<SPHSystem>(fluidParticles, boundaryParticles, pSolver, spaceSize, sphCellLength, sphSmoothingRadius,
                                              dt, sphM0, sphRho0, sphRhoBoundary, sphStiff, sphVisc, sphSurfaceTensionIntensity,
                                              sphAirPressure, sphG, cellSize, bodies, openB);
        if (!pSystem->openBoundariesActive()) { std::fprintf(stderr, "sph_headless: the open boundaries were refused\n"); return 4; }
    } else if (!bodies.empty()) {
        pSystem = std::make_shared<SPHSystem>(fluidParticles, boundaryParticles, pSolver, spaceSize, sphCellLength, sphSmoothingRadius,
                                              dt, sphM0, sphRho0, sphRhoBoundary, sphStiff, sphVisc, sphSurfaceTensionIntensity,
                                              sphAirPressure, sphG, cellSize, bodies);
    } else {
        pSystem = std::make_shared<SPHSystem>(fluidParticles, boundaryParticles, pSolver, spaceSize, sphCellLength, sphSmoothingRadius,
                                              dt, sphM0, sphRho0, sphRhoBoundary, sphStiff, sphVisc, sphSurfaceTensionIntensity,
                                              sphAirPressure, sphG, cellSize);
    }
    if (cudaDeviceSynchronize() != cudaSuccess) {
        std::fprintf(stderr, "sph_headless: %s\n", cudaGetErrorString(cudaGetLastError()));
        return 4;
    }

    if (o.vorticity > 0.0f) basicSolver->setVorticityConfinement(o.vorticity);
    if (o.implicitNu > 0.0f) basicSolver->setImplicitViscosity(o.implicitNu, o.implicitNu);
    if (!o.rheology.empty()) {
        sphb200::Rheology r;
        rheology_of(o, r);
        if (!basicSolver->setRheology(r, o.noSlip ? 1.0f : 0.0f)) {
            std::fprintf(stderr, "sph_headless: --rheology %s was refused\n", o.rheology.c_str());
            return 4;
        }
    }
    if (!o.heat.empty()) {
        sphb200::Thermal t;
        sphb200::ThermalViscosity tv;
        thermal_of(o, t, tv);
        if (!basicSolver->setThermal(t) || (!o.thermalVisc.empty() && !basicSolver->setThermalViscosity(tv))) {
            std::fprintf(stderr, "sph_headless: --heat %s was refused\n", o.heat.c_str());
            return 4;
        }
    }
    if (!o.adhesion.empty()) {
        sphb200::Adhesion a;
        adhesion_of(o, !bodies.empty(), a);
        if (!basicSolver->setAdhesion(a)) {
            std::fprintf(stderr, "sph_headless: --adhesion %s was refused\n", o.adhesion.c_str());
            return 4;
        }
    }
    if (o.tank()) {
        sphb200::TankMotion m;
        tank_of(o, o.box, m);
        if (!pSystem->setTankMotion(m)) {
            std::fprintf(stderr, "sph_headless: the --tank-* motion was refused\n");
            return 4;
        }
    }
    if (o.cfl > 0.0f && !pSystem->setAdaptiveTimeStep(o.cfl, o.dtMin)) {
        std::fprintf(stderr, "sph_headless: --cfl %g --dt-min %g was refused\n", o.cfl, o.dtMin);
        return 4;
    }
    std::FILE* probeCsv = nullptr;
    long long probeLastStep = 0;              // the last step written (the constructor's step 0 is not recorded)
    if (!o.probeOut.empty()) {
        sphb200::Probes p;
        probes_of(o, p);
        // one frame is one step, or with --cfl at most ceil(dt / dt_min) substeps plus the two shortened ones at its end
        const double dtMin = o.dtMin > 0.0f ? o.dtMin : dt / 64.0;
        p.capacity = o.cfl > 0.0f ? static_cast<int>(std::min(65536.0, std::ceil(dt / dtMin) + 2.0)) : 1;
        if (!pSystem->setProbes(p)) { std::fprintf(stderr, "sph_headless: --probe / --gauge were refused\n"); return 4; }
        // a resumed run appends the rows of its frames to the CSV of the run it continues
        probeCsv = std::fopen(o.probeOut.c_str(), o.resume.empty() ? "w" : "a");
        if (!probeCsv) { std::fprintf(stderr, "sph_headless: cannot write --probe-out %s\n", o.probeOut.c_str()); return 5; }
        static const char* kFields[SPHK_PROBE_FIELDS] = {"S", "rho", "vx", "vy", "vz", "p", "T", "n"};
        if (o.resume.empty()) {
            std::fprintf(probeCsv, "step,t");
            for (size_t k = 0; k < p.points.size(); ++k)
                for (const char* f : kFields) std::fprintf(probeCsv, ",p%zu_%s", k, f);
            for (size_t k = 0; k < p.gauges.size(); ++k) std::fprintf(probeCsv, ",g%zu_level", k);
            std::fprintf(probeCsv, "\n");
        }
    }
    // --resume: the state and the frame index (the user section: a little-endian int64)
    int resumedFrom = -1, checkpointsWritten = 0;
    if (!o.resume.empty()) {
        std::vector<unsigned char> user;
        long long frame = -1;
        if (!pSystem->restore(o.resume, &user) || user.size() != sizeof(frame)) {
            std::fprintf(stderr, "sph_headless: --resume %s was refused\n", o.resume.c_str());
            return 4;
        }
        std::memcpy(&frame, user.data(), sizeof(frame));
        if (frame < 0 || frame > o.frames) {
            std::fprintf(stderr, "sph_headless: --resume %s holds frame %lld, outside [0, --frames %d]\n", o.resume.c_str(), frame, o.frames);
            return 4;
        }
        resumedFrom = static_cast<int>(frame);
    }
    auto saveCheckpoint = [&](int frame) {
        const long long f = frame;
        std::vector<unsigned char> user(sizeof(f));
        std::memcpy(user.data(), &f, sizeof(f));
        if (!pSystem->checkpoint(o.checkpoint, user)) return false;
        ++checkpointsWritten;
        return true;
    };
    // the rows recorded since the last drain, one CSV line per step (floats with 9 significant digits: the float32 bits round-trip)
    auto drainProbes = [&]() {
        if (!probeCsv) return;
        const sphb200::ProbeSeries ps = pSystem->probeSeries();
        const size_t nr = static_cast<size_t>(ps.probes) * SPHK_PROBE_FIELDS, ng = static_cast<size_t>(ps.gauges);
        for (size_t r = 0; r < ps.steps.size(); ++r) {
            if (ps.steps[r] <= probeLastStep) continue;
            std::fprintf(probeCsv, "%lld,%.17g", ps.steps[r], ps.times[r]);
            for (size_t k = 0; k < nr; ++k) std::fprintf(probeCsv, ",%.9g", ps.records[r * nr + k]);
            for (size_t k = 0; k < ng; ++k) std::fprintf(probeCsv, ",%.9g", ps.levels[r * ng + k]);
            std::fprintf(probeCsv, "\n");
            probeLastStep = ps.steps[r];
        }
    };

    if (o.bullets > 0) {
        const int hit = slab ? shoot(o, sphSpacing, dt, pSlab->getFluids(), static_cast<size_t>(pSlab->ownedBegin()), static_cast<size_t>(pSlab->size()))
                             : shoot(o, sphSpacing, dt, pSystem->getFluids(), 0, pSystem->getFluids()->size());
        if (hit < 0 || (!slab && hit != o.bullets)) { std::fprintf(stderr, "sph_headless: --bullets found %d of %d particles\n", hit, o.bullets); return 5; }
        if (!slab) pSystem->refreshSpeedBound();   // the shot particles set the first adaptive dt
    }

    // ---- oneStep(), main.cpp:300-306 ----
    int frameId = resumedFrom > 0 ? resumedFrom : 0, straysRouted = 0;
    const int firstFrame = frameId;
    float totalTime = 0.0f, worst = 0.0f;
    std::string substepsJson;
    for (; frameId < o.frames;) {
        ++frameId;
        float milliseconds = 0.0f;
        if (o.cfl > 0.0f) {                              // one frame = dt of simulated time in CFL substeps
            cudaEvent_t e0, e1;
            cudaEventCreate(&e0); cudaEventCreate(&e1);
            cudaEventRecord(e0, pSystem->engine()->stream());
            const int k = pSystem->advance(dt);
            cudaEventRecord(e1, pSystem->engine()->stream());
            cudaEventSynchronize(e1);
            cudaEventElapsedTime(&milliseconds, e0, e1);
            cudaEventDestroy(e0); cudaEventDestroy(e1);
            substepsJson += (substepsJson.empty() ? "" : ", ") + std::to_string(k);
            if (!o.quiet) std::printf("Frame %d - %d substeps, min dt %g s\n", frameId, k, pSystem->adaptiveStats().frameMinDt);
            if (k == 0) return 4;
        } else try {
            milliseconds = slab ? pSlab->step() : pSystem->step();
        } catch (const std::exception& e) {             // SlabSPHSystem::step: a broken decomposition contract ends the rank
            std::fprintf(stderr, "sph_headless: %s\n", e.what());
            std::fflush(nullptr);
            _exit(4);
        }
        if (slab && o.bullets > 0) straysRouted += pSlab->straysRouted();
        drainProbes();
        if (!o.checkpoint.empty() && ((o.checkpointEvery > 0 && frameId % o.checkpointEvery == 0) || frameId == o.frames) &&
            !saveCheckpoint(frameId)) {
            std::fprintf(stderr, "sph_headless: --checkpoint %s was refused\n", o.checkpoint.c_str());
            return 4;
        }
        totalTime += milliseconds;
        worst = milliseconds > worst ? milliseconds : worst;
        if (!o.quiet && !o.heat.empty()) {
            const sphb200::ThermalStats ts = basicSolver->lastThermalStats();
            const int nf = static_cast<int>(pSystem->getFluids()->size());
            std::printf("Frame %d heat - T min %g max %g mean %g, heat %.9g, %d substeps, %d above the stability bound\n", frameId,
                        ts.Tmin, ts.Tmax, nf > 0 ? ts.heat / (double(kSphM0) * nf) : 0.0, ts.heat, ts.substeps, ts.violators);
        }
        if (!o.quiet && !o.adhesion.empty()) {
            const sphb200::AdhesionStats as = basicSolver->lastAdhesionStats();
            std::printf("Frame %d adhesion - %d wetted particles, max acceleration %g m/s^2\n", frameId, as.wetted, as.maxAccel);
        }
        if (!o.quiet && o.tank()) {
            const sphb200::TankState ts = pSystem->tankState();
            std::printf("Frame %d tank - theta %g rad, a_w (%g, %g, %g) m/s^2\n", frameId, ts.theta, ts.accel.x, ts.accel.y, ts.accel.z);
        }
        if (!o.quiet && !o.rheology.empty()) {
            const sphb200::RheologyStats rs = basicSolver->lastRheologyStats();
            std::printf("Frame %d rheology - %d iterations, residual %.3g, max shear rate %g 1/s, %d particles at nu_max\n", frameId,
                        rs.iterations, rs.residual, rs.gammaMax, rs.atNuMax);
        }
        if (!o.quiet)
            std::printf("Frame %d - %2.2f ms, avg time - %2.2f ms/frame (%3.2f FPS)\r", frameId % 10000, milliseconds,
                        totalTime / float(frameId - firstFrame), float(frameId - firstFrame) * 1000.0f / totalTime);
    }
    if (!o.checkpoint.empty() && frameId == firstFrame && !saveCheckpoint(frameId)) {      // (no frame ran: the state as built)
        std::fprintf(stderr, "sph_headless: --checkpoint %s was refused\n", o.checkpoint.c_str());
        return 4;
    }
    if (!o.checkpoint.empty() && !pSystem->waitCheckpoint()) {
        std::fprintf(stderr, "sph_headless: writing --checkpoint %s failed\n", o.checkpoint.c_str());
        return 5;
    }
    if (!o.quiet) std::printf("\n");
    if (probeCsv && std::fclose(probeCsv) != 0) { std::fprintf(stderr, "sph_headless: writing --probe-out %s failed\n", o.probeOut.c_str()); return 5; }

    // ---- optional dump through the public accessors + the render hook (vbo.cu:46-51) ----
    if (!o.dump.empty() && slab) {
        // the particles this rank owns: [ownedBegin, ownedBegin + size) of the local set
        const auto fluids = pSlab->getFluids();
        const size_t n = static_cast<size_t>(pSlab->size()), b = static_cast<size_t>(pSlab->ownedBegin());
        std::vector<float> pos(3 * n), den(n);
        const bool ok = cudaMemcpy(pos.data(), fluids->getPosPtr() + b, n * sizeof(float3), cudaMemcpyDeviceToHost) == cudaSuccess &&
                        cudaMemcpy(den.data(), fluids->getDensityPtr() + b, n * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess &&
                        write_floats(o.dump + ".rank" + std::to_string(o.rank) + ".pos.f32", pos) &&
                        write_floats(o.dump + ".rank" + std::to_string(o.rank) + ".density.f32", den);
        if (!ok) { std::fprintf(stderr, "sph_headless: dump to '%s.rank%d.*' failed\n", o.dump.c_str(), o.rank); return 5; }
    } else if (!o.dump.empty()) {
        const auto fluids = pSystem->getFluids();
        const size_t n = fluids->size();
        std::vector<float> pos(3 * n), den(n), col(3 * n);
        float3 *dDot = nullptr, *dCol = nullptr;
        bool ok = cudaMalloc(&dDot, n * sizeof(float3)) == cudaSuccess && cudaMalloc(&dCol, n * sizeof(float3)) == cudaSuccess;
        if (ok) {
            generate_dots(dDot, dCol, fluids);
            ok = cudaMemcpy(pos.data(), dDot, n * sizeof(float3), cudaMemcpyDeviceToHost) == cudaSuccess &&
                 cudaMemcpy(col.data(), dCol, n * sizeof(float3), cudaMemcpyDeviceToHost) == cudaSuccess &&
                 cudaMemcpy(den.data(), fluids->getDensityPtr(), n * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess;
        }
        cudaFree(dDot); cudaFree(dCol);
        ok = ok && write_floats(o.dump + ".pos.f32", pos) && write_floats(o.dump + ".rgb.f32", col) && write_floats(o.dump + ".density.f32", den);
        if (!ok) { std::fprintf(stderr, "sph_headless: dump to '%s.*' failed\n", o.dump.c_str()); return 5; }
    }
    const float avg = frameId > firstFrame ? totalTime / float(frameId - firstFrame) : 0.0f;
    if (slab) {
        std::printf("{\"solver\": \"%s\", \"rank\": %d, \"ranks\": %d, \"n_fluid\": %d, \"n_owned\": %d, \"halo\": \"%s\", \"strays_routed\": %d, \"dt\": %g, "
                    "\"frames\": %d, \"avg_ms_per_frame\": %.4f, \"max_ms_per_frame\": %.4f}\n",
                    o.solver.c_str(), o.rank, o.ranks, nFluid, pSlab->size(), pSlab->haloTransport(), straysRouted, dt, frameId, avg, worst);
        std::fflush(stdout);
        return 0;
    }
    std::string openJson;
    if (!o.checkpoint.empty() || !o.resume.empty())
        openJson += ", \"resumed_from_frame\": " + std::to_string(resumedFrom) + ", \"checkpoints_written\": " + std::to_string(checkpointsWritten);
    if (o.cfl > 0.0f) {
        const sphb200::AdaptiveStats st = pSystem->adaptiveStats();
        char buf[160];
        std::snprintf(buf, sizeof buf, ", \"simulated_time\": %.17g, \"dt_min_clamps\": %lld, \"nonfinite_steps\": %lld, \"last_dt\": %.9g",
                      pSystem->simulatedTime(), st.minClamps, st.nonFiniteSteps, pSystem->lastTimeStep());
        openJson += ", \"frame_substeps\": [" + substepsJson + "]" + buf;
    }
    if (!o.adhesion.empty()) {
        const sphb200::AdhesionStats as = basicSolver->lastAdhesionStats();
        char buf[96];
        std::snprintf(buf, sizeof buf, ", \"adhesion_wetted\": %d, \"adhesion_max_accel\": %.9g", as.wetted, as.maxAccel);
        openJson += buf;
        if (o.floating) {
            float3 c, J, H;
            float4 q;
            pSystem->getBodyPose(0, c, q);
            pSystem->getBodyImpulse(0, J, H);
            char bb[192];
            std::snprintf(bb, sizeof bb, ", \"body_position\": [%.9g, %.9g, %.9g], \"body_impulse\": [%.9g, %.9g, %.9g]", c.x, c.y, c.z,
                          J.x, J.y, J.z);
            openJson += bb;
        }
    }
    if (!o.meshBody.empty()) {
        float3 c, V, W, J, H;
        float4 q;
        pSystem->getBodyPose(0, c, q);
        pSystem->getBodyMotion(0, V, W);
        pSystem->getBodyImpulse(0, J, H);
        char bb[512];
        std::snprintf(bb, sizeof bb, ", \"body_pose\": [%.9g, %.9g, %.9g, %.9g, %.9g, %.9g, %.9g], \"body_motion\": [%.9g, %.9g, %.9g, %.9g, %.9g, "
                      "%.9g], \"body_impulse\": [%.9g, %.9g, %.9g, %.9g, %.9g, %.9g]", c.x, c.y, c.z, q.x, q.y, q.z, q.w, V.x, V.y, V.z, W.x, W.y,
                      W.z, J.x, J.y, J.z, H.x, H.y, H.z);
        openJson += bb;
    }
    if (open) {
        const sphb200::OpenBoundaryStats st = pSystem->openBoundaryStats();
        openJson += ", \"fluid_count\": " + std::to_string(pSystem->fluidSize()) + ", \"emitted\": " + std::to_string(st.emitted) +
                   ", \"removed\": " + std::to_string(st.removed) + ", \"refused\": " + std::to_string(st.refused) +
                   ", \"open_check\": " + std::to_string(pSystem->openBoundaryCheck());
    }
    std::printf("{\"solver\": \"%s\", \"n_fluid\": %d, \"n_boundary\": %d, \"cells\": [%d, %d, %d], \"dt\": %g, \"frames\": %d, "
                "\"avg_ms_per_frame\": %.4f, \"max_ms_per_frame\": %.4f, \"particle_steps_per_s\": %.1f%s}\n",
                o.solver.c_str(), nFluid, nBoundary, cellSize.x, cellSize.y, cellSize.z, dt, frameId, avg, worst,
                avg > 0.0f ? double(nFluid) / (double(avg) * 1e-3) : 0.0, openJson.c_str());
    return 0;
}
