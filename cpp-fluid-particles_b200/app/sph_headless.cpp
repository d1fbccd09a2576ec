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
//                [--cfl C [--dt-min X]]
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
    float cfl = 0.0f;                         // --cfl C: CFL-adaptive substeps, --dt of simulated time per frame (0: off)
    float dtMin = 0.0f;                       // --dt-min X: their smallest dt (0: dt / 64)
    int bullets = 0;                          // test aid: this many top-layer particles start at ~3 cell planes per step
    int ranks = 1, rank = -1;                 // --ranks N: SlabSPHSystem on N GPUs; --rank R: this process is rank R
    std::string rendezvous;
};

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
        else if (a == "--cfl" && need(i, 1)) o.cfl = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--dt-min" && need(i, 1)) o.dtMin = static_cast<float>(std::atof(argv[++i]));
        else if (a == "--ranks" && need(i, 1)) o.ranks = std::atoi(argv[++i]);
        else if (a == "--rank" && need(i, 1)) o.rank = std::atoi(argv[++i]);
        else if (a == "--rendezvous" && need(i, 1)) o.rendezvous = argv[++i];
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
    if (!(o.cfl >= 0.0f) || !std::isfinite(o.cfl) || !(o.dtMin >= 0.0f) || !std::isfinite(o.dtMin)) {
        std::fprintf(stderr, "sph_headless: --cfl C and --dt-min X need finite values > 0\n");
        return false;
    }
    if (o.cfl > 0.0f && o.ranks > 1) {
        std::fprintf(stderr, "sph_headless: --cfl runs on one GPU only (adaptive time stepping is not supported with --ranks)\n");
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
                             "[--tap SPEED] [--drain SIDE] [--capacity N] [--cfl C [--dt-min X]] [--dump PREFIX] [--quiet] [--emit-scene PREFIX] "
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
    std::vector<sphb200::KinematicBody> bodies;
    std::vector<float3> fluidPoints = fluid_block(o, sphSpacing);
    if (o.stir) bodies.push_back(paddle(o, sphSpacing, boundarySpacing));
    if (o.floating) bodies.push_back(floating_cube(o, sphSpacing, boundarySpacing));
    if (!bodies.empty()) fluidPoints = clear_of(fluidPoints, bodies[0], boundarySpacing);
    const sphb200::OpenBoundaries openB = open_boundaries(o, sphSpacing);
    const bool open = !openB.emitters.empty() || !openB.sinks.empty();
    if (!o.emitScene.empty()) {
        const int3 cells = cellSize;
        bool ok = write_floats(o.emitScene + ".fluid.f32", flat(fluidPoints)) &&
                  write_floats(o.emitScene + ".boundary.f32", flat(boundary_shell(cells, spaceSize)));
        if (ok && !bodies.empty()) {
            const auto& b = bodies[0];
            ok = write_floats(o.emitScene + ".body.f32", flat(b.points)) &&
                 write_floats(o.emitScene + ".body_state.f32",
                              {b.position.x, b.position.y, b.position.z, b.orientation.x, b.orientation.y, b.orientation.z, b.orientation.w,
                               b.linearVelocity.x, b.linearVelocity.y, b.linearVelocity.z, b.angularVelocity.x, b.angularVelocity.y,
                               b.angularVelocity.z});
            if (ok && o.floating)
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
    auto boundaryParticles = std::make_shared<SPHParticles>(boundary_shell(cellSize, spaceSize));
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
    if (o.cfl > 0.0f && !pSystem->setAdaptiveTimeStep(o.cfl, o.dtMin)) {
        std::fprintf(stderr, "sph_headless: --cfl %g --dt-min %g was refused\n", o.cfl, o.dtMin);
        return 4;
    }

    if (o.bullets > 0) {
        const int hit = slab ? shoot(o, sphSpacing, dt, pSlab->getFluids(), static_cast<size_t>(pSlab->ownedBegin()), static_cast<size_t>(pSlab->size()))
                             : shoot(o, sphSpacing, dt, pSystem->getFluids(), 0, pSystem->getFluids()->size());
        if (hit < 0 || (!slab && hit != o.bullets)) { std::fprintf(stderr, "sph_headless: --bullets found %d of %d particles\n", hit, o.bullets); return 5; }
        if (!slab) pSystem->refreshSpeedBound();   // the shot particles set the first adaptive dt
    }

    // ---- oneStep(), main.cpp:300-306 ----
    int frameId = 0, straysRouted = 0;
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
        totalTime += milliseconds;
        worst = milliseconds > worst ? milliseconds : worst;
        if (!o.quiet)
            std::printf("Frame %d - %2.2f ms, avg time - %2.2f ms/frame (%3.2f FPS)\r", frameId % 10000, milliseconds,
                        totalTime / float(frameId), float(frameId) * 1000.0f / totalTime);
    }
    if (!o.quiet) std::printf("\n");

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
    const float avg = frameId ? totalTime / float(frameId) : 0.0f;
    if (slab) {
        std::printf("{\"solver\": \"%s\", \"rank\": %d, \"ranks\": %d, \"n_fluid\": %d, \"n_owned\": %d, \"halo\": \"%s\", \"strays_routed\": %d, \"dt\": %g, "
                    "\"frames\": %d, \"avg_ms_per_frame\": %.4f, \"max_ms_per_frame\": %.4f}\n",
                    o.solver.c_str(), o.rank, o.ranks, nFluid, pSlab->size(), pSlab->haloTransport(), straysRouted, dt, frameId, avg, worst);
        std::fflush(stdout);
        return 0;
    }
    std::string openJson;
    if (o.cfl > 0.0f) {
        const sphb200::AdaptiveStats st = pSystem->adaptiveStats();
        char buf[160];
        std::snprintf(buf, sizeof buf, ", \"simulated_time\": %.17g, \"dt_min_clamps\": %lld, \"nonfinite_steps\": %lld, \"last_dt\": %.9g",
                      pSystem->simulatedTime(), st.minClamps, st.nonFiniteSteps, pSystem->lastTimeStep());
        openJson += ", \"frame_substeps\": [" + substepsJson + "]" + buf;
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
