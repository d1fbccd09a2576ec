// sph_app.cpp -- headless facade; see include/sph_app.h.
//
// Restates the reference's API call sites (main.cpp:86,117 particle construction; :119-130 solver
// construction; :131-134 SPHSystem construction; :302 step; vbo.cu:48 accessor use) and nothing
// else.  It is deliberately written ONLY against names the reference headers export, so that it
// builds unchanged on top of either engine (this repo's headers, or /root/reference/src).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <iostream>
#include <vector>
#include <memory>
#include <cuda_runtime.h>
#ifdef SPH_APP_REFERENCE_ENGINE
#include <helper_math.h>
#include "global.h"
#endif
#include "DArray.h"
#include "Particles.h"
#include "SPHParticles.h"
#include "BaseSolver.h"
#include "BasicSPHSolver.h"
#include "DFSPHSolver.h"
#include "PBDSolver.h"
#include "SPHSystem.h"
#include "sph_app.h"

// One batch in flight through the pipelined host-buffer path (sph_app_submit / sph_app_wait)
struct sph_batch {
    float3* dIn[2] = {nullptr, nullptr};     // device staging: pos, vel of the batch
    float3* dOut[2] = {nullptr, nullptr};    // device staging of the result: pos, vel
    float* dOutDensity = nullptr;
    cudaEvent_t uploaded = nullptr, computed = nullptr, downloaded = nullptr;
    float* hPos = nullptr; float* hVel = nullptr; float* hDensity = nullptr;   // where the result goes (host)
    bool pending = false;                    // uploaded, not yet stepped
    float ms = 0.f;
};

struct sph_app {
    std::shared_ptr<SPHSystem> system;
    BaseSolver* solver = nullptr;            // owned by `system` (its constructor moves the caller's shared_ptr)
    // pipelined path (created on first sph_app_submit): uploads and downloads on their own streams (PCIe is full duplex)
    cudaStream_t copyStream = nullptr, downStream = nullptr;
    sph_batch batch[2];
    unsigned long long submitted = 0;
    bool pipeReady = false;
    ~sph_app() {
        if (pipeReady) {
            cudaStreamSynchronize(copyStream);
            cudaStreamSynchronize(downStream);
            for (auto& b : batch) {
                cudaFree(b.dIn[0]); cudaFree(b.dIn[1]); cudaFree(b.dOut[0]); cudaFree(b.dOut[1]); cudaFree(b.dOutDensity);
                cudaEventDestroy(b.uploaded); cudaEventDestroy(b.computed); cudaEventDestroy(b.downloaded);
            }
            cudaStreamDestroy(copyStream);
            cudaStreamDestroy(downStream);
        }
    }
};

static std::vector<float3> to_float3(const float* xyz, int n) {
    std::vector<float3> v(static_cast<size_t>(n));
    for (int i = 0; i < n; ++i) v[i] = make_float3(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]);
    return v;
}

#ifdef SPH_APP_REFERENCE_ENGINE
struct body_list {};
struct open_list {};
#else
using body_list = std::vector<sphb200::KinematicBody>;
using open_list = sphb200::OpenBoundaries;
#endif

// open: emitters and sinks with a fluid capacity of max_fluid (nullptr: a closed system of n_fluid particles)
static sph_app* create(const float* fluid_xyz, int n_fluid, const float* boundary_xyz, int n_boundary, const sph_app_params* p,
                       const body_list* bodies, const open_list* open = nullptr, int max_fluid = 0) {
    if (!fluid_xyz || !boundary_xyz || !p || n_fluid <= 0 || n_boundary <= 0) return nullptr;
#ifdef SPH_APP_REFERENCE_ENGINE
    auto fluidParticles = std::make_shared<SPHParticles>(to_float3(fluid_xyz, n_fluid));
    const int num = static_cast<int>(fluidParticles->size());
#else
    auto fluidParticles = open ? std::make_shared<SPHParticles>(to_float3(fluid_xyz, n_fluid), static_cast<unsigned int>(max_fluid))
                               : std::make_shared<SPHParticles>(to_float3(fluid_xyz, n_fluid));
    const int num = static_cast<int>(fluidParticles->capacity());
#endif
    auto boundaryParticles = std::make_shared<SPHParticles>(to_float3(boundary_xyz, n_boundary));
    std::shared_ptr<BaseSolver> pSolver;
    switch (p->solver) {
    case 2:
        if (p->max_iter > 0) pSolver = std::make_shared<PBDSolver>(num, p->max_iter);
        else pSolver = std::make_shared<PBDSolver>(num);
        break;
    case 1:
        if (p->max_iter > 0)
            pSolver = std::make_shared<DFSPHSolver>(num, p->density_error_threshold,
                                                    p->divergence_error_threshold, p->max_iter);
        else pSolver = std::make_shared<DFSPHSolver>(num);
        break;
    default:
        pSolver = std::make_shared<BasicSPHSolver>(num);
        break;
    }
    auto* app = new sph_app;
    app->solver = pSolver.get();
    const float3 space = make_float3(p->space[0], p->space[1], p->space[2]), G = make_float3(p->gravity[0], p->gravity[1], p->gravity[2]);
    const int3 cells = make_int3(p->cell_size[0], p->cell_size[1], p->cell_size[2]);
#ifndef SPH_APP_REFERENCE_ENGINE
    if (open)
        app->system = std::make_shared<SPHSystem>(fluidParticles, boundaryParticles, pSolver, space, p->cell_length, p->radius, p->dt,
                                                  p->m0, p->rho0, p->rho_boundary, p->stiff, p->visc, p->surface_tension,
                                                  p->air_pressure, G, cells, body_list{}, *open);
    else if (bodies)
        app->system = std::make_shared<SPHSystem>(fluidParticles, boundaryParticles, pSolver, space, p->cell_length, p->radius, p->dt,
                                                  p->m0, p->rho0, p->rho_boundary, p->stiff, p->visc, p->surface_tension,
                                                  p->air_pressure, G, cells, *bodies);
    else
#endif
        app->system = std::make_shared<SPHSystem>(fluidParticles, boundaryParticles, pSolver, space, p->cell_length, p->radius, p->dt,
                                                  p->m0, p->rho0, p->rho_boundary, p->stiff, p->visc, p->surface_tension,
                                                  p->air_pressure, G, cells);
    (void)bodies; (void)open; (void)max_fluid;
    if (cudaDeviceSynchronize() != cudaSuccess) {
        std::fprintf(stderr, "sph_app_create: %s\n", cudaGetErrorString(cudaGetLastError()));
        delete app;
        return nullptr;
    }
    return app;
}

extern "C" sph_app* sph_app_create(const float* fluid_xyz, int n_fluid, const float* boundary_xyz, int n_boundary,
                                   const sph_app_params* p) {
    return create(fluid_xyz, n_fluid, boundary_xyz, n_boundary, p, nullptr);
}

#ifndef SPH_APP_REFERENCE_ENGINE
// the bodies of sph_app_create_with_bodies / _with_dynamic_bodies (mass_inertia: null = all kinematic)
static sph_app* create_with_bodies(const float* fluid_xyz, int n_fluid, const float* boundary_xyz, int n_boundary, int n_bodies,
                                   const int* body_begin, const float* body_xyz, const float* pose, const float* motion,
                                   const float* mass_inertia, const sph_app_params* p) {
    if (n_bodies < 0 || (n_bodies > 0 && (!body_begin || !body_xyz || !pose || !motion)) || (n_bodies > 0 && body_begin[0] != 0))
        return nullptr;
    body_list bodies(static_cast<size_t>(n_bodies));
    bool dynamic = false;
    for (int b = 0; b < n_bodies; ++b) {
        if (body_begin[b + 1] < body_begin[b]) return nullptr;
        auto& k = bodies[b];
        k.points = to_float3(body_xyz + 3 * static_cast<size_t>(body_begin[b]), body_begin[b + 1] - body_begin[b]);
        const float* P = pose + 7 * b;
        const float* M = motion + 6 * b;
        k.position = make_float3(P[0], P[1], P[2]);
        k.orientation = make_float4(P[3], P[4], P[5], P[6]);
        k.linearVelocity = make_float3(M[0], M[1], M[2]);
        k.angularVelocity = make_float3(M[3], M[4], M[5]);
        if (mass_inertia) {
            const float* D = mass_inertia + 4 * b;
            k.mass = D[0];
            k.inertia = make_float3(D[1], D[2], D[3]);
            dynamic = dynamic || D[0] > 0.0f;
        }
    }
    sph_app* app = create(fluid_xyz, n_fluid, boundary_xyz, n_boundary, p, &bodies);
    // sphk_bodies_init or sphk_bodies_set_dynamics refused them
    if (app && (app->system->bodyCount() != n_bodies || app->system->bodiesDynamic() != dynamic)) { delete app; return nullptr; }
    return app;
}
#endif

extern "C" sph_app* sph_app_create_with_bodies(const float* fluid_xyz, int n_fluid, const float* boundary_xyz, int n_boundary,
                                               int n_bodies, const int* body_begin, const float* body_xyz, const float* pose,
                                               const float* motion, const sph_app_params* p) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)fluid_xyz; (void)n_fluid; (void)boundary_xyz; (void)n_boundary; (void)n_bodies; (void)body_begin; (void)body_xyz;
    (void)pose; (void)motion; (void)p;
    return nullptr;
#else
    return create_with_bodies(fluid_xyz, n_fluid, boundary_xyz, n_boundary, n_bodies, body_begin, body_xyz, pose, motion, nullptr, p);
#endif
}

extern "C" sph_app* sph_app_create_with_dynamic_bodies(const float* fluid_xyz, int n_fluid, const float* boundary_xyz,
                                                       int n_boundary, int n_bodies, const int* body_begin, const float* body_xyz,
                                                       const float* pose, const float* motion, const float* mass_inertia,
                                                       const sph_app_params* p) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)fluid_xyz; (void)n_fluid; (void)boundary_xyz; (void)n_boundary; (void)n_bodies; (void)body_begin; (void)body_xyz;
    (void)pose; (void)motion; (void)mass_inertia; (void)p;
    return nullptr;
#else
    if (!mass_inertia) return nullptr;
    return create_with_bodies(fluid_xyz, n_fluid, boundary_xyz, n_boundary, n_bodies, body_begin, body_xyz, pose, motion,
                              mass_inertia, p);
#endif
}

extern "C" sph_app* sph_app_create_open(const float* fluid_xyz, int n_fluid, int max_fluid, const float* boundary_xyz, int n_boundary,
                                        int n_emitters, const sph_app_emitter* emitters, int n_sinks, const float* sinks_lo_hi,
                                        const sph_app_params* p) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)fluid_xyz; (void)n_fluid; (void)max_fluid; (void)boundary_xyz; (void)n_boundary; (void)n_emitters; (void)emitters;
    (void)n_sinks; (void)sinks_lo_hi; (void)p;
    return nullptr;
#else
    if (max_fluid < n_fluid || n_emitters < 0 || n_sinks < 0 || (n_emitters > 0 && !emitters) || (n_sinks > 0 && !sinks_lo_hi))
        return nullptr;
    open_list open;
    for (int k = 0; k < n_emitters; ++k) {
        const sph_app_emitter& e = emitters[k];
        sphb200::Emitter m;
        m.origin = make_float3(e.origin[0], e.origin[1], e.origin[2]);
        m.direction = make_float3(e.direction[0], e.direction[1], e.direction[2]);
        m.speed = e.speed; m.spacing = e.spacing; m.width = e.width; m.height = e.height;
        open.emitters.push_back(m);
    }
    for (int k = 0; k < n_sinks; ++k) {
        const float* b = sinks_lo_hi + 6 * k;
        open.sinks.push_back({make_float3(b[0], b[1], b[2]), make_float3(b[3], b[4], b[5])});
    }
    sph_app* app = create(fluid_xyz, n_fluid, boundary_xyz, n_boundary, p, nullptr, &open, max_fluid);
    // the class layer refused them (it then builds the closed system)
    if (app && (n_emitters > 0 || n_sinks > 0) && !app->system->openBoundariesActive()) { delete app; return nullptr; }
    return app;
#endif
}

extern "C" int sph_app_open_boundary_stats(sph_app* app, long long* stats3, int* check_bits) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)stats3; (void)check_bits;
    return 1;
#else
    if (!app) return 1;
    const sphb200::OpenBoundaryStats s = app->system->openBoundaryStats();
    if (stats3) { stats3[0] = s.emitted; stats3[1] = s.removed; stats3[2] = s.refused; }
    if (check_bits) *check_bits = app->system->openBoundaryCheck();
    return 0;
#endif
}

extern "C" int sph_app_set_body_motion(sph_app* app, int body, const float* linear_velocity, const float* angular_velocity) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)body; (void)linear_velocity; (void)angular_velocity;
    return 1;
#else
    if (!app || !linear_velocity || !angular_velocity || body < 0 || body >= app->system->bodyCount()) return 1;
    for (int a = 0; a < 3; ++a)
        if (!std::isfinite(linear_velocity[a]) || !std::isfinite(angular_velocity[a])) return 1;
    app->system->setBodyMotion(body, make_float3(linear_velocity[0], linear_velocity[1], linear_velocity[2]),
                               make_float3(angular_velocity[0], angular_velocity[1], angular_velocity[2]));
    return 0;
#endif
}

extern "C" int sph_app_body_pose(sph_app* app, int body, float* pose) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)body; (void)pose;
    return 1;
#else
    if (!app || !pose || body < 0 || body >= app->system->bodyCount()) return 1;
    float3 c;
    float4 q;
    app->system->getBodyPose(body, c, q);
    const float v[7] = {c.x, c.y, c.z, q.x, q.y, q.z, q.w};
    std::copy(v, v + 7, pose);
    return 0;
#endif
}

static int body_pair(sph_app* app, int body, float* out, bool impulse) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)body; (void)out; (void)impulse;
    return 1;
#else
    if (!app || !out || body < 0 || body >= app->system->bodyCount()) return 1;
    float3 a, b;
    if (impulse) app->system->getBodyImpulse(body, a, b);
    else app->system->getBodyMotion(body, a, b);
    const float v[6] = {a.x, a.y, a.z, b.x, b.y, b.z};
    std::copy(v, v + 6, out);
    return 0;
#endif
}

extern "C" int sph_app_body_motion(sph_app* app, int body, float* motion) { return body_pair(app, body, motion, false); }

extern "C" int sph_app_body_impulse(sph_app* app, int body, float* impulse) { return body_pair(app, body, impulse, true); }

extern "C" void sph_app_destroy(sph_app* app) { delete app; }

extern "C" float sph_app_step(sph_app* app) { return app->system->step(); }

extern "C" int sph_app_fluid_size(const sph_app* app) { return app->system->fluidSize(); }
extern "C" int sph_app_boundary_size(const sph_app* app) { return app->system->boundarySize(); }

static int d2h(void* dst, const void* src, size_t bytes) {
    if (!dst) return 0;
    return cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : 1;
}

extern "C" int sph_app_download_fluid(sph_app* app, float* pos, float* vel, float* density,
                                      float* pressure, float* mass, int* p2c) {
    const auto f = app->system->getFluids();
    const size_t n = f->size();
    int bad = 0;
    bad |= d2h(pos, f->getPosPtr(), n * sizeof(float3));
    bad |= d2h(vel, f->getVelPtr(), n * sizeof(float3));
    bad |= d2h(density, f->getDensityPtr(), n * sizeof(float));
    bad |= d2h(pressure, f->getPressurePtr(), n * sizeof(float));
    bad |= d2h(mass, f->getMassPtr(), n * sizeof(float));
    bad |= d2h(p2c, f->getParticle2Cell(), n * sizeof(int));
    return bad;
}

extern "C" int sph_app_download_boundary(sph_app* app, float* pos, float* mass, int* p2c) {
    const auto b = app->system->getBoundaries();
    const size_t n = b->size();
    int bad = 0;
    bad |= d2h(pos, b->getPosPtr(), n * sizeof(float3));
    bad |= d2h(mass, b->getMassPtr(), n * sizeof(float));
    bad |= d2h(p2c, b->getParticle2Cell(), n * sizeof(int));
    return bad;
}

extern "C" int sph_app_upload_fluid(sph_app* app, const float* pos, const float* vel) {
    const auto f = app->system->getFluids();
    const size_t n = f->size();
    int bad = 0;
    if (pos) bad |= cudaMemcpy(f->getPosPtr(), pos, n * sizeof(float3), cudaMemcpyHostToDevice) != cudaSuccess;
    if (vel) bad |= cudaMemcpy(f->getVelPtr(), vel, n * sizeof(float3), cudaMemcpyHostToDevice) != cudaSuccess;
#ifndef SPH_APP_REFERENCE_ENGINE
    app->system->refreshSpeedBound();       // an adaptive system's next dt sees the uploaded state
#endif
    return bad;
}

// ---- pipelined host-buffer stepping -------------------------------------------------------------------------------
// The reference's own call sites move data with synchronous cudaMemcpy through the raw accessors (Particles.h:24,
// vbo.cu:48).  A caller that feeds a batch of particle states from host memory and reads every result back pays
// ~2 ms of PCIe time per 2M-particle step that way.  sph_app_submit overlaps those copies with the previous batch's
// step: uploads and downloads run on a copy stream into / out of device staging buffers, the step itself only adds
// two device-to-device copies.  Only public accessors and the CUDA runtime are used, so this builds on either engine.
static bool pipe_init(sph_app* app) {
    if (app->pipeReady) return true;
    const size_t n = app->system->getFluids()->size();
    if (cudaStreamCreateWithFlags(&app->copyStream, cudaStreamNonBlocking) != cudaSuccess) return false;
    if (cudaStreamCreateWithFlags(&app->downStream, cudaStreamNonBlocking) != cudaSuccess) return false;
    for (auto& b : app->batch) {
        bool ok = true;
        for (int k = 0; k < 2; ++k) {
            ok = ok && cudaMalloc(reinterpret_cast<void**>(&b.dIn[k]), n * sizeof(float3)) == cudaSuccess;
            ok = ok && cudaMalloc(reinterpret_cast<void**>(&b.dOut[k]), n * sizeof(float3)) == cudaSuccess;
        }
        ok = ok && cudaMalloc(reinterpret_cast<void**>(&b.dOutDensity), n * sizeof(float)) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&b.uploaded, cudaEventDisableTiming) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&b.computed, cudaEventDisableTiming) == cudaSuccess;
        ok = ok && cudaEventCreateWithFlags(&b.downloaded, cudaEventDisableTiming) == cudaSuccess;
        ok = ok && cudaEventRecord(b.downloaded, app->downStream) == cudaSuccess;      // "nothing to wait for" before the first use
        if (!ok) return false;
    }
    app->pipeReady = true;
    return true;
}

// steps the batch in `slot` (its upload has been enqueued) and enqueues the download of its result
static int pipe_run(sph_app* app, int slot) {
    sph_batch& b = app->batch[slot];
    if (!b.pending) return 0;
    const auto f = app->system->getFluids();
    const size_t n = f->size();
    int bad = 0;
    // legacy default stream: ordered with everything the engines enqueue (the reference uses it throughout; this
    // repository's engine stream is a blocking stream)
    bad |= cudaStreamWaitEvent(nullptr, b.uploaded, 0) != cudaSuccess;
    bad |= cudaMemcpyAsync(f->getPosPtr(), b.dIn[0], n * sizeof(float3), cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess;
    bad |= cudaMemcpyAsync(f->getVelPtr(), b.dIn[1], n * sizeof(float3), cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess;
    b.ms = app->system->step();
    bad |= cudaStreamWaitEvent(nullptr, b.downloaded, 0) != cudaSuccess;     // this slot's previous result has left the staging buffers
    bad |= cudaMemcpyAsync(b.dOut[0], f->getPosPtr(), n * sizeof(float3), cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess;
    bad |= cudaMemcpyAsync(b.dOut[1], f->getVelPtr(), n * sizeof(float3), cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess;
    bad |= cudaMemcpyAsync(b.dOutDensity, f->getDensityPtr(), n * sizeof(float), cudaMemcpyDeviceToDevice, nullptr) != cudaSuccess;
    bad |= cudaEventRecord(b.computed, nullptr) != cudaSuccess;
    bad |= cudaStreamWaitEvent(app->downStream, b.computed, 0) != cudaSuccess;
    if (b.hPos) bad |= cudaMemcpyAsync(b.hPos, b.dOut[0], n * sizeof(float3), cudaMemcpyDeviceToHost, app->downStream) != cudaSuccess;
    if (b.hVel) bad |= cudaMemcpyAsync(b.hVel, b.dOut[1], n * sizeof(float3), cudaMemcpyDeviceToHost, app->downStream) != cudaSuccess;
    if (b.hDensity) bad |= cudaMemcpyAsync(b.hDensity, b.dOutDensity, n * sizeof(float), cudaMemcpyDeviceToHost, app->downStream) != cudaSuccess;
    bad |= cudaEventRecord(b.downloaded, app->downStream) != cudaSuccess;
    b.pending = false;
    return bad;
}

extern "C" int sph_app_submit(sph_app* app, const float* pos_in, const float* vel_in, float* pos_out, float* vel_out,
                              float* density_out) {
    if (!app || !pos_in || !vel_in) return 1;
#ifndef SPH_APP_REFERENCE_ENGINE
    if (app->system->openBoundariesActive()) return 1;      // the pipelining assumes a fixed particle count
    if (app->system->adaptiveTimeStep()) return 1;          // ... and a fixed step
#endif
    if (!pipe_init(app)) return 1;
    const size_t n = app->system->getFluids()->size();
    const int slot = static_cast<int>(app->submitted & 1ull);
    sph_batch& b = app->batch[slot];
    int bad = 0;
    // (the slot's previous batch was stepped during the previous submit, so its input staging is free; its download reads
    // the output staging, which this batch overwrites only after ITS step and after waiting for the `downloaded` event)
    bad |= cudaMemcpyAsync(b.dIn[0], pos_in, n * sizeof(float3), cudaMemcpyHostToDevice, app->copyStream) != cudaSuccess;
    bad |= cudaMemcpyAsync(b.dIn[1], vel_in, n * sizeof(float3), cudaMemcpyHostToDevice, app->copyStream) != cudaSuccess;
    bad |= cudaEventRecord(b.uploaded, app->copyStream) != cudaSuccess;
    b.hPos = pos_out; b.hVel = vel_out; b.hDensity = density_out;
    b.pending = true;
    app->submitted++;
    // while this upload is in flight, step the batch submitted before it
    bad |= pipe_run(app, slot ^ 1);
    return bad;
}

extern "C" int sph_app_wait(sph_app* app) {
    if (!app || !app->pipeReady) return 0;
    int bad = 0;
    const int last = static_cast<int>((app->submitted + 1) & 1ull);     // slot of the most recent submit
    bad |= pipe_run(app, last ^ 1);
    bad |= pipe_run(app, last);
    bad |= cudaStreamSynchronize(app->copyStream) != cudaSuccess;
    bad |= cudaStreamSynchronize(app->downStream) != cudaSuccess;
    return bad;
}

// ---- introspection of this repository's engine (absent from the reference build of the facade) -------------------------
extern "C" int sph_app_dfsph_iterations(sph_app* app, int* divergence_iters, int* density_iters) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)divergence_iters; (void)density_iters;
    return 1;
#else
    auto* d = dynamic_cast<DFSPHSolver*>(app->solver);
    if (!d) return 1;
    if (divergence_iters) *divergence_iters = d->lastDivergenceIterations();
    if (density_iters) *density_iters = d->lastDensityIterations();
    return 0;
#endif
}

extern "C" int sph_app_set_option(sph_app* app, int option, int value) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)option; (void)value;
    return 1;
#else
    switch (option) {
    case 1: { auto* d = dynamic_cast<DFSPHSolver*>(app->solver); if (!d) return 1; d->setDeviceLoops(value != 0); return 0; }
    case 2: { auto* b = dynamic_cast<BasicSPHSolver*>(app->solver); if (!b) return 1; b->setFusedSweeps(value != 0); return 0; }
    case 3: app->system->setStepGraph(value != 0); return 0;
    default: return 1;
    }
#endif
}

extern "C" int sph_app_step_graph_active(sph_app* app) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app;
    return -1;
#else
    return app->system->stepGraphActive() ? 1 : 0;
#endif
}

extern "C" int sph_app_set_vorticity(sph_app* app, float eps) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)eps;
    return 1;
#else
    auto* b = dynamic_cast<BasicSPHSolver*>(app->solver);
    if (!b || !(eps >= 0.0f)) return 1;
    b->setVorticityConfinement(eps);
    return 0;
#endif
}

extern "C" int sph_app_set_implicit_viscosity(sph_app* app, float nu, float nu_boundary, float tol, int max_iter) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)nu; (void)nu_boundary; (void)tol; (void)max_iter;
    return 1;
#else
    auto* b = dynamic_cast<BasicSPHSolver*>(app->solver);
    if (!b || !(nu >= 0.0f) || !(nu_boundary >= 0.0f) || !std::isfinite(nu) || !std::isfinite(nu_boundary) || !(tol > 0.0f) ||
        max_iter < 1 || max_iter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER)
        return 1;
    if (nu_boundary > 0.0f && app->system->bodiesDynamic()) return 1;   // the viscous wall force is not part of the bodies' reaction
    b->setImplicitViscosity(nu, nu_boundary, tol, max_iter);
    return 0;
#endif
}

extern "C" int sph_app_viscosity_stats(sph_app* app, int* iterations, float* rel_residual) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)iterations; (void)rel_residual;
    return 1;
#else
    auto* b = dynamic_cast<BasicSPHSolver*>(app->solver);
    if (!b) return 1;
    if (iterations) *iterations = b->lastViscosityIterations();
    if (rel_residual) *rel_residual = b->lastViscosityResidual();
    return 0;
#endif
}

extern "C" int sph_app_set_adaptive_dt(sph_app* app, float C, float dt_min, float dt_max) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)C; (void)dt_min; (void)dt_max;
    return 1;
#else
    if (!app) return 1;
    if (C == 0.0f) { app->system->disableAdaptiveTimeStep(); return 0; }
    return app->system->setAdaptiveTimeStep(C, dt_min, dt_max) ? 0 : 1;
#endif
}

extern "C" int sph_app_advance(sph_app* app, double frame_seconds, int* substeps, float* min_dt) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)frame_seconds; (void)substeps; (void)min_dt;
    return 1;
#else
    if (!app || !app->system->adaptiveTimeStep() || !(frame_seconds > 0.0) || !std::isfinite(frame_seconds)) return 1;
    const int k = app->system->advance(frame_seconds);
    if (substeps) *substeps = k;
    if (min_dt) *min_dt = app->system->adaptiveStats().frameMinDt;
    return k > 0 ? 0 : 1;
#endif
}

extern "C" int sph_app_adaptive_stats(sph_app* app, float* speed_dt3, int* source, long long* counts2, double* simulated_time) {
#ifdef SPH_APP_REFERENCE_ENGINE
    (void)app; (void)speed_dt3; (void)source; (void)counts2; (void)simulated_time;
    return 1;
#else
    if (!app) return 1;
    const sphb200::AdaptiveStats s = app->system->adaptiveStats();
    if (speed_dt3) { speed_dt3[0] = s.speed; speed_dt3[1] = app->system->lastTimeStep(); speed_dt3[2] = s.frameMinDt; }
    if (source) *source = s.source;
    if (counts2) { counts2[0] = s.minClamps; counts2[1] = s.nonFiniteSteps; }
    if (simulated_time) *simulated_time = app->system->simulatedTime();
    return 0;
#endif
}

extern "C" const char* sph_app_engine(void) {
#ifdef SPH_APP_REFERENCE_ENGINE
    return "reference-cuda";
#else
    return "b200-native";
#endif
}
