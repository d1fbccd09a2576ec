// sph_api.cpp -- host-side orchestration of one simulation step over the libsphk C-ABI.
// Each method states the reference code whose behaviour it reproduces (/root/reference/src/...).
// No device code here: this file is compiled by g++.
#include "sph_api.hpp"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>

using sphb200::check;

// the checkpoint checksum of host bytes (the config record's hashes)
static unsigned long long stateHash(const void* p, unsigned long long bytes) {
    unsigned long long h = 0;
    check(sphk_state_checksum_host(p, bytes, &h), "sphk_state_checksum_host");
    return h;
}

// ================================================================================================
// Engine
// ================================================================================================
namespace sphb200 {
Engine::Engine(int maxFluid, int maxBoundary, int3 cellSize, float cellLength, int3 origin) {
    // blocking stream: legacy-default-stream work of the caller (DArray memset, cudaMemcpy through the
    // raw accessors) orders with the engine's work exactly as it does in the single-stream reference
    CUDA_CALL(cudaStreamCreate(&stream_));
    sphk_grid g;
    g.cell_size[0] = cellSize.x; g.cell_size[1] = cellSize.y; g.cell_size[2] = cellSize.z;
    g.cell_length = cellLength;
    g.origin[0] = origin.x; g.origin[1] = origin.y; g.origin[2] = origin.z;
    const int rc = sphk_create(&ctx_, maxFluid, maxBoundary, &g, stream_);
    if (rc != 0) {
        // no CPU fallback: a missing device / failed allocation is reported and leaves the system inert
        printf("sphk_create failed: %s (%d)\n", sphk_error_string(rc), rc);
        ctx_ = nullptr;
    }
}
Engine::~Engine() {
    if (ctx_) { sphk_synchronize(ctx_); sphk_destroy(ctx_); }
    if (stream_) cudaStreamDestroy(stream_);
}
}  // namespace sphb200

// ================================================================================================
// Particles (Particles.h:22-25, Particles.cu:28-36)
// ================================================================================================
Particles::Particles(const std::vector<float3>& p) : pos(p.size()), vel(p.size()) {
    CUDA_CALL(cudaMemcpy(pos.addr(), p.data(), sizeof(float3) * p.size(), cudaMemcpyHostToDevice));
}

Particles::Particles(const std::vector<float3>& p, unsigned int capacity)
    : pos(std::max<size_t>(capacity, p.size())), vel(std::max<size_t>(capacity, p.size())), activeCount_(static_cast<int>(p.size())) {
    CUDA_CALL(cudaMemcpy(pos.addr(), p.data(), sizeof(float3) * p.size(), cudaMemcpyHostToDevice));
}

void Particles::advect(float dt) {
    // pos += dt * vel.  Not on the engine's hot path (BasicSPHSolver::advect uses the fused sphk_advect); kept for
    // API parity.  It moves particles behind the engine's back, so the packed records are re-packed before the
    // next sweep (shadowsStale).
    cudaStream_t st = nullptr;
    if (engine_ && engine_->ok()) { st = engine_->stream(); engine_->shadowsStale = true; }
    check(sphk_particles_advect(reinterpret_cast<float*>(pos.addr()), reinterpret_cast<const float*>(vel.addr()),
                                static_cast<int>(size()), dt, st), "sphk_particles_advect");
}

// ================================================================================================
// BasicSPHSolver (BasicSPHSolver.cu)
// ================================================================================================
bool BasicSPHSolver::beginStep(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                               const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float radius,
                               bool neighborList, int listSkinPermille) {
    const auto& eng = fluids->engine();
    if (!eng || !eng->ok()) {
        printf("SPH solver: particles are not bound to an engine (construct them through SPHSystem)\n");
        current_.ctx = nullptr;
        return false;
    }
    current_.ctx = eng->ctx();
    current_.abi.fluid = fluids->abi();
    current_.abi.boundary = boundaries->abi();
    current_.abi.cell_start_fluid = cellStartFluid.addr();
    current_.abi.cell_start_boundary = cellStartBoundary.addr();
    current_.abi.radius = radius;
    reacting_ = eng->bodiesDynamic;
    bodies_ = eng->bodies;
    check(sphk_set_option(current_.ctx, SPHK_OPT_NEIGHBOR_LIST, neighborList ? 1 : 0), "sphk_set_option");
    check(sphk_set_option(current_.ctx, SPHK_OPT_LIST_SKIN, listSkinPermille), "sphk_set_option");
    if (eng->shadowsStale) { check(sphk_refresh(current_.ctx, &current_.abi), "sphk_refresh"); eng->shadowsStale = false; }
    // the temperatures follow their particles through the search of this step (once per search, like the solvers' history arrays)
    if (thermalOn_) check(sphk_permute(current_.ctx, temperature_->addr(), 1, static_cast<int>(fluids->size())), "sphk_permute");
    return true;
}

// BasicSPHSolver::step, BasicSPHSolver.cu:237-260
void BasicSPHSolver::step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                          const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                          int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float stiff,
                          float visc, float3 G, float surfaceTensionIntensity, float airPressure) {
    if (!beginStep(fluids, boundaries, cellStartFluid, cellStartBoundary, radius, true, 0)) return;
    force(fluids, dt, G);
    if (fusedSweeps_) {
        // density and the colour gradient depend on positions and masses only: one sweep computes both, before the velocity
        // terms (the reference computes them in two sweeps, :277-330 and :32-83, with nothing in between that they read)
        if (surfaceTensionIntensity > EPSILON || airPressure > EPSILON) {
            check(sphk_fused_density_color_grad(current_.ctx, &current_.abi, colorGradBuffer(), rho0, rhoB), "sphk_fused_density_color_grad");
            produced(0, colorGradBuffer(), 3);
        } else {
            check(sphk_density(current_.ctx, &current_.abi), "sphk_density");
        }
    }
    velocityStage(fluids, boundaries, cellStartFluid, cellStartBoundary, cellSize, cellLength, radius, rho0, rhoB, visc, dt,
                  surfaceTensionIntensity, airPressure, false, G);
    if (fusedSweeps_) {
        check(sphk_pressure(current_.ctx, &current_.abi, rho0, stiff), "sphk_pressure");
        produced(0, fluids->getDensityPtr(), 1); produced(0, fluids->getPressurePtr(), 1);
        check(sphk_pressure_force(current_.ctx, &current_.abi, dt), "sphk_pressure_force");
        react(-dt);
    } else {
        project(fluids, boundaries, cellStartFluid, cellStartBoundary, rho0, stiff, cellSize, cellLength, radius, dt);
    }
    advect(fluids, dt, spaceSize);
}

// The velocity terms every solver applies between its density and its pressure (PBD: after its position) solve.  Fused sweeps
// where the library has them; one sweep per reference launch site through the virtual hooks otherwise, and where there is nothing
// to fuse (PBD's XSPH through its diffuse override).
void BasicSPHSolver::velocityStage(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                                   const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, int3 cellSize,
                                   float cellLength, float radius, float rho0, float rhoB, float visc, float dt,
                                   float surfaceTensionIntensity, float airPressure, bool xsph, float3 G) {
    const bool surface = surfaceTensionIntensity > EPSILON || airPressure > EPSILON;
    float* dv = reinterpret_cast<float*>(bufferFloat3.addr());
    float* cg = colorGradBuffer();
    if (fusedSweeps_ && xsph && (surface || vorticityOn())) {
        // XSPH + colour gradient (positions are final after the projection) + omega from the velocities XSPH reads, in one sweep
        if (vorticityOn()) {
            check(sphk_fused_pbd_xsph_vorticity(current_.ctx, &current_.abi, visc, rho0, surface ? cg : nullptr, rhoB, omegaBuffer(),
                                                omegaNormBuffer()),
                  "sphk_fused_pbd_xsph_vorticity");
            producedVel(fluids); produced(2, omegaNormBuffer(), 1);
        } else {
            check(sphk_fused_pbd_xsph_color_grad(current_.ctx, &current_.abi, visc, rho0, cg, rhoB), "sphk_fused_pbd_xsph_color_grad");
            producedVel(fluids);
        }
        if (surface) {
            produced(0, cg, 3);
            check(sphk_surface(current_.ctx, &current_.abi, cg, dt, rho0, surfaceTensionIntensity, airPressure), "sphk_surface");
            producedVel(fluids);
        }
    } else if (fusedSweeps_ && !xsph && surface) {
        // viscosity + surface from the colour gradient of the density sweep (+ omega from the velocities the viscosity term reads)
        if (vorticityOn()) {
            check(sphk_fused_viscosity_surface_vorticity(current_.ctx, &current_.abi, dv, cg, rho0, visc, dt, surfaceTensionIntensity,
                                                         airPressure, omegaBuffer(), omegaNormBuffer()),
                  "sphk_fused_viscosity_surface_vorticity");
            produced(2, omegaNormBuffer(), 1);
        } else {
            check(sphk_fused_viscosity_surface(current_.ctx, &current_.abi, dv, cg, rho0, visc, dt, surfaceTensionIntensity, airPressure),
                  "sphk_fused_viscosity_surface");
        }
        producedVel(fluids);
    } else {
        if (vorticityOn()) vorticity(rho0);
        diffuse(fluids, cellStartFluid, cellSize, cellLength, rho0, radius, visc, dt);
        producedVel(fluids);
        if (surface)
            handleSurface(fluids, boundaries, cellStartFluid, cellStartBoundary, rho0, rhoB, cellSize, cellLength, radius,
                          dt, surfaceTensionIntensity, airPressure);
    }
    if (adhesionOn_) {
        check(sphk_adhesion(current_.ctx, &current_.abi, &adhesionAbi_, dt, rho0, rhoB), "sphk_adhesion");
        producedVel(fluids);
    }
    if (rheoOn_) rheology(fluids, rho0, rhoB, dt);        // replaces the constant-nu solve
    else if (thermalOn_ && thermalViscOn_) thermalViscosity(fluids, rho0, rhoB, dt);
    else if (implicitViscosityOn()) implicitViscosity(fluids, rho0, rhoB, dt);
    if (vorticityOn()) confine(fluids, rho0, dt);
    if (thermalOn_) heat(fluids, rho0, rhoB, dt, G);
}

// addition (no reference counterpart): vorticity confinement, sphk.h
void BasicSPHSolver::setVorticityConfinement(float eps) {
    if (!(eps >= 0.0f)) {
        printf("setVorticityConfinement: eps must be >= 0 (got %g); the setting is kept at %g\n", eps, vortEps_);
        return;
    }
    if (eps > 0.0f && !omega_) {
        omega_ = std::make_unique<DArray<float3>>(num_);
        omegaNorm_ = std::make_unique<DArray<float>>(num_);
    }
    if (eps != vortEps_) ++configEpoch_;
    vortEps_ = eps;
}

void BasicSPHSolver::vorticity(float rho0) {
    check(sphk_vorticity(current_.ctx, &current_.abi, omegaBuffer(), omegaNormBuffer(), rho0), "sphk_vorticity");
    produced(2, omegaNormBuffer(), 1);
}

void BasicSPHSolver::confine(const std::shared_ptr<SPHParticles>& fluids, float rho0, float dt) {
    check(sphk_vorticity_confinement(current_.ctx, &current_.abi, omegaBuffer(), omegaNormBuffer(), vortEps_, dt, rho0),
          "sphk_vorticity_confinement");
    producedVel(fluids);
}

// addition (no reference counterpart): implicit viscosity, sphk.h
void BasicSPHSolver::setImplicitViscosity(float nu, float nuBoundary, float tol, int maxIter) {
    if (!(nu >= 0.0f) || !(nuBoundary >= 0.0f) || !(tol > 0.0f) || maxIter < 1 || maxIter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER ||
        !std::isfinite(nu) || !std::isfinite(nuBoundary)) {
        printf("setImplicitViscosity: need nu >= 0, nuBoundary >= 0 (finite), tol > 0 and 1 <= maxIter <= %d (got %g, %g, %g, %d); "
               "the setting is kept at %g, %g, %g, %d\n", SPHK_IMPLICIT_VISCOSITY_MAX_ITER, nu, nuBoundary, tol, maxIter, implNu_,
               implNuB_, implTol_, implMaxIter_);
        return;
    }
    if (nuBoundary > 0.0f && reacting_) {      // (known once the solver has stepped in its system: SPHSystem's constructor does)
        printf("setImplicitViscosity: nuBoundary > 0 is not supported with dynamic bodies (the viscous wall force is not part of "
               "their reaction); the setting is kept at %g, %g, %g, %d\n", implNu_, implNuB_, implTol_, implMaxIter_);
        return;
    }
    if (nu > 0.0f && !viscWork_)
        viscWork_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(sphk_implicit_viscosity_work_floats(num_)));
    if (nu != implNu_ || nuBoundary != implNuB_ || tol != implTol_ || maxIter != implMaxIter_) ++configEpoch_;
    implNu_ = nu; implNuB_ = nuBoundary; implTol_ = tol; implMaxIter_ = maxIter;
}

void BasicSPHSolver::implicitViscosity(const std::shared_ptr<SPHParticles>& fluids, float rho0, float rhoB, float dt) {
    check(sphk_implicit_viscosity(current_.ctx, &current_.abi, viscWork_->addr(), implNu_, implNuB_, dt, rho0, rhoB, implTol_,
                                  implMaxIter_),
          "sphk_implicit_viscosity");
    producedVel(fluids);
}

void BasicSPHSolver::viscStats(int& iters, float& residual) const {
    iters = 0; residual = 0.0f;
    if (current_.ctx) check(sphk_implicit_viscosity_stats(current_.ctx, &iters, &residual), "sphk_implicit_viscosity_stats");
}
int BasicSPHSolver::lastViscosityIterations() const { int it; float r; viscStats(it, r); return it; }
float BasicSPHSolver::lastViscosityResidual() const { int it; float r; viscStats(it, r); return r; }

// addition (no reference counterpart): non-Newtonian viscosity, sphk.h
static bool rheologyValid(const sphb200::Rheology& r) {
    for (float p : r.params) if (!std::isfinite(p)) return false;
    if (!std::isfinite(r.nu_min) || !std::isfinite(r.nu_max) || !(r.nu_min >= 0.0f) || r.nu_min > r.nu_max) return false;
    const float* p = r.params;
    if (r.model == SPHK_RHEOLOGY_CROSS) return p[0] >= 0.0f && p[1] >= 0.0f && p[2] >= 0.0f && p[3] > 0.0f;
    if (r.model == SPHK_RHEOLOGY_HERSCHEL_BULKLEY) return p[0] >= 0.0f && p[1] > 0.0f && p[2] >= 0.0f && p[3] >= 0.0f;
    return false;
}

bool BasicSPHSolver::setRheology(const sphb200::Rheology& r, float boundaryFactor, float tol, int maxIter) {
    if (!rheologyValid(r) || !(boundaryFactor >= 0.0f) || !std::isfinite(boundaryFactor) || !(tol > 0.0f) || maxIter < 1 ||
        maxIter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER) {
        printf("setRheology: need a known model with finite parameters in range, 0 <= nuMin <= nuMax (finite), boundaryFactor >= 0, "
               "tol > 0 and 1 <= maxIter <= %d; the setting is kept\n", SPHK_IMPLICIT_VISCOSITY_MAX_ITER);
        return false;
    }
    if (thermalViscOn_) {
        printf("setRheology: not together with a temperature-dependent viscosity; the setting is kept\n");
        return false;
    }
    if (boundaryFactor > 0.0f && reacting_) {
        printf("setRheology: boundaryFactor > 0 is not supported with dynamic bodies (the viscous wall force is not part of their "
               "reaction); the setting is kept\n");
        return false;
    }
    if (!rheoWork_)
        rheoWork_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(sphk_rheology_work_floats(num_)));
    viscosityField();
    if (!rheoOn_ || std::memcmp(&r, &rheo_, sizeof(sphk_rheology)) != 0 || boundaryFactor != rheoBeta_ || tol != rheoTol_ ||
        maxIter != rheoMaxIter_)
        ++configEpoch_;
    rheoOn_ = true; rheo_ = r; rheoBeta_ = boundaryFactor; rheoTol_ = tol; rheoMaxIter_ = maxIter;
    return true;
}

void BasicSPHSolver::clearRheology() {
    if (rheoOn_) ++configEpoch_;
    rheoOn_ = false;
}

const DArray<float>& BasicSPHSolver::viscosityField() const {
    if (!nuField_) nuField_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(num_));
    return *nuField_;
}

void BasicSPHSolver::rheology(const std::shared_ptr<SPHParticles>& fluids, float rho0, float rhoB, float dt) {
    check(sphk_non_newtonian_viscosity(current_.ctx, &current_.abi, rheoWork_->addr(), nuField_->addr(), &rheo_, rheoBeta_, dt, rho0,
                                       rhoB, rheoTol_, rheoMaxIter_),
          "sphk_non_newtonian_viscosity");
    producedVel(fluids);
}

sphb200::RheologyStats BasicSPHSolver::lastRheologyStats() const {
    sphb200::RheologyStats s;
    if (current_.ctx)
        check(sphk_non_newtonian_stats(current_.ctx, &s.iterations, &s.residual, &s.gammaMax, &s.nuMin, &s.nuMax, &s.atNuMax),
              "sphk_non_newtonian_stats");
    return s;
}

// addition (no reference counterpart): heat transfer, sphk.h
static bool finiteNonneg(float x) { return std::isfinite(x) && x >= 0.0f; }

bool BasicSPHSolver::setThermal(const sphb200::Thermal& t) {
    bool ok = finiteNonneg(t.alpha) && std::isfinite(t.beta) && std::isfinite(t.Tref) && std::isfinite(t.wall.T) && finiteNonneg(t.wall.h) &&
              t.bodies.size() <= SPHK_BODY_LIMIT;
    for (const auto& g : t.bodies) ok = ok && std::isfinite(g.T) && finiteNonneg(g.h);
    for (float T : t.emitterT) ok = ok && std::isfinite(T);
    if (!ok) {
        printf("setThermal: need alpha >= 0, finite beta, Tref and temperatures, conductances h >= 0 (finite) and at most %d bodies; "
               "the setting is kept\n", SPHK_BODY_LIMIT);
        return false;
    }
    if (tankOn_) {
        printf("setThermal: not under a tank motion (the Boussinesq buoyancy acts along the constant G); the setting is kept\n");
        return false;
    }
    if (bodies_ >= 0 && static_cast<int>(t.bodies.size()) > bodies_) {
        printf("setThermal: %d body entries, but the system has %d bodies; the setting is kept\n", static_cast<int>(t.bodies.size()),
               bodies_);
        return false;
    }
    if (!temperatureSet_) {
        const std::vector<float> init(static_cast<size_t>(num_), t.Tref);
        CUDA_CALL(cudaMemcpy(temperatureField().addr(), init.data(), sizeof(float) * init.size(), cudaMemcpyHostToDevice));
        temperatureSet_ = true;
    }
    sphk_thermal a{};
    a.alpha = t.alpha; a.beta = t.beta; a.t_ref = t.Tref;
    a.n_groups = 1 + static_cast<int>(t.bodies.size());
    a.groups[0] = {t.wall.T, t.wall.h};
    for (size_t b = 0; b < t.bodies.size(); ++b) a.groups[b + 1] = {t.bodies[b].T, t.bodies[b].h};
    if (!thermalOn_ || std::memcmp(&a, &thermalAbi_, sizeof(a)) != 0) ++configEpoch_;
    thermalOn_ = true; thermal_ = t; thermalAbi_ = a;
    return true;
}

void BasicSPHSolver::clearThermal() {
    if (thermalOn_) ++configEpoch_;
    thermalOn_ = false;
}

DArray<float>& BasicSPHSolver::temperatureField() {
    if (!temperature_) {
        temperature_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(num_));
        heatWork_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(num_));
    }
    return *temperature_;
}

bool BasicSPHSolver::setThermalViscosity(const sphb200::ThermalViscosity& v) {
    if (!finiteNonneg(v.nuRef) || !std::isfinite(v.E) || !finiteNonneg(v.nuMin) || !finiteNonneg(v.nuMax) || v.nuMin > v.nuMax ||
        !finiteNonneg(v.wallFactor) || !(v.tol > 0.0f) || v.maxIter < 1 || v.maxIter > SPHK_IMPLICIT_VISCOSITY_MAX_ITER) {
        printf("setThermalViscosity: need nuRef >= 0, finite E, 0 <= nuMin <= nuMax (finite), wallFactor >= 0, tol > 0 and 1 <= maxIter "
               "<= %d; the setting is kept\n", SPHK_IMPLICIT_VISCOSITY_MAX_ITER);
        return false;
    }
    if (rheoOn_) {
        printf("setThermalViscosity: not together with a shear-rate rheology; the setting is kept\n");
        return false;
    }
    if (v.wallFactor > 0.0f && reacting_) {
        printf("setThermalViscosity: wallFactor > 0 is not supported with dynamic bodies (the viscous wall force is not part of their "
               "reaction); the setting is kept\n");
        return false;
    }
    if (!viscWork_)
        viscWork_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(sphk_implicit_viscosity_work_floats(num_)));
    viscosityField();
    if (!thermalViscOn_ || std::memcmp(&v, &thermalVisc_, sizeof(v)) != 0) ++configEpoch_;
    thermalViscOn_ = true; thermalVisc_ = v;
    return true;
}

void BasicSPHSolver::clearThermalViscosity() {
    if (thermalViscOn_) ++configEpoch_;
    thermalViscOn_ = false;
}

void BasicSPHSolver::thermalViscosity(const std::shared_ptr<SPHParticles>& fluids, float rho0, float rhoB, float dt) {
    const sphb200::ThermalViscosity& v = thermalVisc_;
    const sphk_viscosity_law law{v.nuRef, v.E, thermal_.Tref, v.nuMin, v.nuMax};
    check(sphk_thermal_viscosity(current_.ctx, &current_.abi, viscWork_->addr(), nuField_->addr(), temperature_->addr(), &law,
                                 v.wallFactor, dt, rho0, rhoB, v.tol, v.maxIter),
          "sphk_thermal_viscosity");
    producedVel(fluids);
}

void BasicSPHSolver::heat(const std::shared_ptr<SPHParticles>& fluids, float rho0, float rhoB, float dt, float3 G) {
    int k = 1;
    check(sphk_heat_substeps(&thermalAbi_, current_.abi.radius, dt, &k), "sphk_heat_substeps");
    heatSubsteps_ = k;
    const float g[3] = {G.x, G.y, G.z};
    for (int j = 0; j < k; ++j)
        check(sphk_heat_step(current_.ctx, &current_.abi, &thermalAbi_, temperature_->addr(), heatWork_->addr(), dt, j, k, rho0, rhoB, g),
              "sphk_heat_step");
    producedVel(fluids);
}

sphb200::ThermalStats BasicSPHSolver::lastThermalStats() {
    sphb200::ThermalStats s;
    s.substeps = heatSubsteps_;
    if (current_.ctx && temperature_)
        check(sphk_heat_stats(current_.ctx, temperature_->addr(), current_.abi.fluid.mass, current_.abi.fluid.n, &s.maxCourant,
                              &s.violators, &s.Tmin, &s.Tmax, &s.heat),
              "sphk_heat_stats");
    return s;
}

// addition (no reference counterpart): fluid-solid adhesion, sphk.h
bool BasicSPHSolver::setAdhesion(const sphb200::Adhesion& a) {
    bool ok = finiteNonneg(a.wall) && a.bodies.size() <= SPHK_BODY_LIMIT;
    for (float b : a.bodies) ok = ok && finiteNonneg(b);
    if (!ok) {
        printf("setAdhesion: need finite beta >= 0 and at most %d bodies; the setting is kept\n", SPHK_BODY_LIMIT);
        return false;
    }
    if (bodies_ >= 0 && static_cast<int>(a.bodies.size()) > bodies_) {
        printf("setAdhesion: %d body entries, but the system has %d bodies; the setting is kept\n", static_cast<int>(a.bodies.size()),
               bodies_);
        return false;
    }
    sphk_adhesion_setting abi{};
    abi.n_groups = 1 + static_cast<int>(a.bodies.size());
    abi.beta[0] = a.wall;
    for (size_t b = 0; b < a.bodies.size(); ++b) abi.beta[b + 1] = a.bodies[b];
    if (!adhesionOn_ || std::memcmp(&abi, &adhesionAbi_, sizeof(abi)) != 0) ++configEpoch_;
    adhesionOn_ = true; adhesionAbi_ = abi;
    return true;
}

void BasicSPHSolver::clearAdhesion() {
    if (adhesionOn_) ++configEpoch_;
    adhesionOn_ = false;
}

sphb200::AdhesionStats BasicSPHSolver::lastAdhesionStats() const {
    sphb200::AdhesionStats s;
    if (current_.ctx) check(sphk_adhesion_stats(current_.ctx, &s.wetted, &s.maxAccel), "sphk_adhesion_stats");
    return s;
}

// :227-235
void BasicSPHSolver::force(std::shared_ptr<SPHParticles>&, float dt, float3 G) {
    if (!current_.ctx) return;
    if (tankOn_) {                  // addition: the tank frame's body force instead of gravity (DESIGN.md section 2.15)
        check(sphk_tank_force(current_.ctx, &current_.abi, dt), "sphk_tank_force");
        return;
    }
    const float g[3] = {G.x, G.y, G.z};
    check(sphk_gravity(current_.ctx, &current_.abi, dt, g), "sphk_gravity");
}

// :98-101
void BasicSPHSolver::advect(std::shared_ptr<SPHParticles>&, float dt, float3 spaceSize) {
    if (!current_.ctx) return;
    const float sp[3] = {spaceSize.x, spaceSize.y, spaceSize.z};
    check(sphk_advect(current_.ctx, &current_.abi, dt, sp), "sphk_advect");
}

// :167-181
void BasicSPHSolver::project(std::shared_ptr<SPHParticles>&, const std::shared_ptr<SPHParticles>&, const DArray<int>&,
                             const DArray<int>&, float rho0, float stiff, int3, float, float, float dt) {
    if (!current_.ctx) return;
    check(sphk_density(current_.ctx, &current_.abi), "sphk_density");
    check(sphk_pressure(current_.ctx, &current_.abi, rho0, stiff), "sphk_pressure");
    produced(0, current_.abi.fluid.density, 1); produced(0, current_.abi.fluid.pressure, 1);
    check(sphk_pressure_force(current_.ctx, &current_.abi, dt), "sphk_pressure_force");
    react(-dt);
}

// :211-225
void BasicSPHSolver::diffuse(std::shared_ptr<SPHParticles>&, const DArray<int>&, int3, float, float rho0, float,
                             float visc, float dt) {
    if (!current_.ctx) return;
    check(sphk_viscosity(current_.ctx, &current_.abi, reinterpret_cast<float*>(bufferFloat3.addr()), rho0, visc, dt),
          "sphk_viscosity");
}

// :262-275
void BasicSPHSolver::handleSurface(std::shared_ptr<SPHParticles>&, const std::shared_ptr<SPHParticles>&,
                                   const DArray<int>&, const DArray<int>&, float rho0, float rhoB, int3, float, float,
                                   float dt, float surfaceTensionIntensity, float airPressure) {
    if (!current_.ctx) return;
    float* cg = reinterpret_cast<float*>(bufferFloat3.addr());
    check(sphk_color_grad(current_.ctx, &current_.abi, cg, rho0, rhoB), "sphk_color_grad");
    produced(0, cg, 3);
    check(sphk_surface(current_.ctx, &current_.abi, cg, dt, rho0, surfaceTensionIntensity, airPressure), "sphk_surface");
    produced(1, current_.abi.fluid.vel, 3);
}

// ================================================================================================
// DFSPHSolver (DFSPHSolver.cu)
// ================================================================================================
// DFSPHSolver::step, DFSPHSolver.cu:33-72
void DFSPHSolver::step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                       const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                       int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float,
                       float visc, float3 G, float surfaceTensionIntensity, float airPressure) {
    if (!beginStep(fluids, boundaries, cellStartFluid, cellStartBoundary, radius, true, 0)) return;
    const int num = static_cast<int>(fluids->size());
    if (fusedSweeps_) {
        // density/alpha + colour gradient (positions only) + the first divergence error of :341 in one sweep
        const bool surface = surfaceTensionIntensity > EPSILON || airPressure > EPSILON;
        check(sphk_fused_dfsph_density_alpha_div_error(current_.ctx, &current_.abi, alpha.addr(), surface ? colorGradBuffer() : nullptr,
                                                       rho0, rhoB, error.addr(), bufferFloat.addr(), dt),
              "sphk_fused_dfsph_density_alpha_div_error");
        produced(2, bufferFloat.addr(), 1);
        if (surface) produced(0, colorGradBuffer(), 3);
    } else {
        check(sphk_dfsph_density_alpha(current_.ctx, &current_.abi, alpha.addr()), "sphk_dfsph_density_alpha");
    }
    itDiv_ = correctDivergenceError(rho0, dt, divergenceErrorThreshold, maxIter, num, fusedSweeps_);
    force(fluids, dt, G);
    velocityStage(fluids, boundaries, cellStartFluid, cellStartBoundary, cellSize, cellLength, radius, rho0, rhoB, visc, dt,
                  surfaceTensionIntensity, airPressure, false, G);
    itDen_ = project(fluids, boundaries, cellStartFluid, cellStartBoundary, rho0, cellSize, cellLength, radius, dt,
                     densityErrorThreshold, maxIter);
    advect(fluids, dt, spaceSize);
}

// DFSPHSolver::correctDivergenceError, DFSPHSolver.cu:331-363.  With a negative threshold the loop test
// `totalError > thr*num*rho0` is true for every possible error sum, so the (host-synchronising)
// reduction is skipped: same iteration count as the reference, no pipeline bubble (Q11).
int DFSPHSolver::correctDivergenceError(float rho0, float dt, float errorThreshold, int maxIter_, int num, bool firstErrorDone) {
    auto totalError = std::numeric_limits<float>::max();
    auto iter = 0;
    sphk_ctx* ctx = current_.ctx;
    if (!firstErrorDone) {
        check(sphk_dfsph_div_error(ctx, &current_.abi, alpha.addr(), error.addr(), bufferFloat.addr(), dt, rho0),
              "sphk_dfsph_div_error");
        produced(2, bufferFloat.addr(), 1);
    }
    const float thresholdCount = static_cast<float>(globalCount_ >= 0 ? globalCount_ : num);
    if (errorThreshold >= 0.0f && deviceLoops_ && !fieldHook_) {
        // the loop test runs on the device: maxIter bodies are enqueued, the ones after convergence return at once
        check(sphk_loop_begin(ctx, 0, 1, maxIter_, errorThreshold * num * rho0, 1), "sphk_loop_begin");
        for (int k = 0; k < maxIter_; ++k) {
            check(sphk_dfsph_div_correct(ctx, &current_.abi, bufferFloat.addr()), "sphk_dfsph_div_correct");
            react(1.0f);
            check(sphk_dfsph_div_error(ctx, &current_.abi, alpha.addr(), error.addr(), bufferFloat.addr(), dt, rho0),
                  "sphk_dfsph_div_error");
            check(sphk_loop_next(ctx, 0, error.addr(), num), "sphk_loop_next");
        }
        check(sphk_loop_end(ctx, 0), "sphk_loop_end");
        return -1;      // known on the device; lastDivergenceIterations() reads it back
    }
    while ((iter < 1 || totalError > errorThreshold * thresholdCount * rho0) && iter < maxIter_) {
        check(sphk_dfsph_div_correct(ctx, &current_.abi, bufferFloat.addr()), "sphk_dfsph_div_correct");
        react(1.0f);
        produced(1, current_.abi.fluid.vel, 3);
        ++iter;
        // After the last permitted iteration the loop ends whatever the error is, and nothing reads this error, stiffness or
        // record scalar again: the density solve forms its own before it reads them.  The reference's final error sweep
        // (DFSPHSolver.cu:354) is dead work -- one of the 20 list sweeps of a fixed 4+4 step.
        if (iter == maxIter_) break;
        check(sphk_dfsph_div_error(ctx, &current_.abi, alpha.addr(), error.addr(), bufferFloat.addr(), dt, rho0),
              "sphk_dfsph_div_error");
        produced(2, bufferFloat.addr(), 1);
        if (errorThreshold >= 0.0f) totalError = reduceError(num);
    }
    return iter;
}

// DFSPHSolver::project, DFSPHSolver.cu:160-210
int DFSPHSolver::project(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>&, const DArray<int>&,
                         const DArray<int>&, float rho0, int3, float, float, float dt, float errorThreshold,
                         int maxIter_) {
    if (!current_.ctx) return 0;
    sphk_ctx* ctx = current_.ctx;
    const int num = static_cast<int>(fluids->size());
    auto totalError = std::numeric_limits<float>::max();
    auto iter = 0;
    // warm stiffness of the previous step follows its particle (:170-171)
    check(sphk_permute(ctx, denWarmStiff.addr(), 1, num), "sphk_permute");
    // (ghost particles carry their warm stiffness with them: it travels with the candidates and is permuted with the rest)
    check(sphk_dfsph_den_correct(ctx, &current_.abi, denWarmStiff.addr(), dt), "sphk_dfsph_den_correct");
    react(1.0f / dt);
    produced(1, current_.abi.fluid.vel, 3);
    check(sphk_dfsph_den_error(ctx, &current_.abi, alpha.addr(), error.addr(), bufferFloat.addr(), dt, rho0, nullptr),
          "sphk_dfsph_den_error");
    produced(2, bufferFloat.addr(), 1);
    check(sphk_copy(ctx, denWarmStiff.addr(), bufferFloat.addr(), num), "sphk_copy");     // :185
    const float thresholdCount = static_cast<float>(globalCount_ >= 0 ? globalCount_ : num);
    if (errorThreshold >= 0.0f && deviceLoops_ && !fieldHook_) {
        check(sphk_loop_begin(ctx, 1, 2, maxIter_, errorThreshold * num * rho0, 2), "sphk_loop_begin");
        for (int k = 0; k < maxIter_; ++k) {
            check(sphk_dfsph_den_correct(ctx, &current_.abi, bufferFloat.addr(), dt), "sphk_dfsph_den_correct");
            react(1.0f / dt);
            check(sphk_dfsph_den_error(ctx, &current_.abi, alpha.addr(), error.addr(), bufferFloat.addr(), dt, rho0,
                                       denWarmStiff.addr()),
                  "sphk_dfsph_den_error");                                                // + :199-203 fused
            check(sphk_loop_next(ctx, 1, error.addr(), num), "sphk_loop_next");
        }
        check(sphk_loop_end(ctx, 1), "sphk_loop_end");
        return -1;
    }
    while ((iter < 2 || totalError > errorThreshold * thresholdCount * rho0) && iter < maxIter_) {
        check(sphk_dfsph_den_correct(ctx, &current_.abi, bufferFloat.addr(), dt), "sphk_dfsph_den_correct");
        react(1.0f / dt);
        produced(1, current_.abi.fluid.vel, 3);
        check(sphk_dfsph_den_error(ctx, &current_.abi, alpha.addr(), error.addr(), bufferFloat.addr(), dt, rho0,
                                   denWarmStiff.addr()),
              "sphk_dfsph_den_error");                                                    // + :199-203 fused
        produced(2, bufferFloat.addr(), 1);
        ++iter;
        if (iter >= 2 && errorThreshold >= 0.0f) totalError = reduceError(num);
    }
    return iter;
}

// thrust::reduce(error, abs_plus), DFSPHSolver.cu:206,360 -- over the particles this rank owns, then over the ranks
float DFSPHSolver::reduceError(int num) {
    float local = 0.0f;
    if (reduceHook_) {
        int begin = 0, count = num;
        if (ownedRange_) ownedRange_(begin, count);
        check(sphk_reduce_abs_sum(current_.ctx, error.addr(begin), count, &local), "sphk_reduce_abs_sum");
        return static_cast<float>(reduceHook_(static_cast<double>(local)));
    }
    check(sphk_reduce_abs_sum(current_.ctx, error.addr(), num, &local), "sphk_reduce_abs_sum");
    return local;
}

int DFSPHSolver::loopIterations(int slot, int hostCount) const {
    if (hostCount >= 0 || !current_.ctx) return hostCount;
    int it = 0;
    check(sphk_loop_iterations(current_.ctx, slot, &it, nullptr), "sphk_loop_iterations");
    return it;
}

// ================================================================================================
// PBDSolver (PBDSolver.cu)
// ================================================================================================
// PBDSolver::step, PBDSolver.cu:34-73
void PBDSolver::step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                     const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                     int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float, float,
                     float3 G, float surfaceTensionIntensity, float airPressure) {
    if (!posLastInitialized) {
        if (fluids->engine() && fluids->engine()->ok()) sphk_synchronize(fluids->engine()->ctx());
        initializePosLast(fluids->getPos());
        throw "PBD: The last position of fluids is initialized.";     // Q6, PBDSolver.cu:44-47
    }
    // positions move inside the step (Q7): the neighbour list carries a skin of 0.15 R; the engine tracks the
    // displacement on the device and falls back to the cell walk if the corrections ever exceed skin/2
    if (!beginStep(fluids, boundaries, cellStartFluid, cellStartBoundary, radius, true, 150)) return;
    updateNeighborhood(fluids);
    // the positions were advanced by the last predict: its dt is the interval of the projection and the velocity derivation
    const float dtPrev = historyTimeStep(dt);
    reactCoef_ = 1.0f / (rho0 * dtPrev);
    project(fluids, boundaries, cellStartFluid, cellStartBoundary, rho0, cellSize, spaceSize, cellLength, radius, maxIter);
    check(sphk_pbd_velocity_from_positions(current_.ctx, &current_.abi, reinterpret_cast<float*>(fluidPosLast.addr()), dtPrev),
          "sphk_pbd_velocity_from_positions");
    velocityStage(fluids, boundaries, cellStartFluid, cellStartBoundary, cellSize, cellLength, radius, rho0, rhoB, xSPH_c, dt,
                  surfaceTensionIntensity, airPressure, true, G);
    force(fluids, dt, G);
    predict(fluids, dt, spaceSize);
}

// :75-79
void PBDSolver::predict(std::shared_ptr<SPHParticles>& fluids, float dt, float3 spaceSize) {
    check(sphk_copy(current_.ctx, reinterpret_cast<float*>(fluidPosLast.addr()),
                    reinterpret_cast<const float*>(fluids->getPosPtr()), 3 * static_cast<int>(fluids->size())),
          "sphk_copy");
    advect(fluids, dt, spaceSize);
    lastPredictDt_ = dt;
}

// :81-87
void PBDSolver::updateNeighborhood(const std::shared_ptr<SPHParticles>& particles) {
    check(sphk_permute(current_.ctx, reinterpret_cast<float*>(fluidPosLast.addr()), 3, static_cast<int>(particles->size())),
          "sphk_permute");
}

// :117-125
void PBDSolver::diffuse(std::shared_ptr<SPHParticles>&, const DArray<int>&, int3, float, float rho0, float, float visc) {
    check(sphk_pbd_xsph(current_.ctx, &current_.abi, visc, rho0), "sphk_pbd_xsph");
}
void PBDSolver::diffuse(std::shared_ptr<SPHParticles>& fluids, const DArray<int>& cellStartFluid, int3 cellSize, float cellLength,
                        float rho0, float radius, float visc, float) {
    diffuse(fluids, cellStartFluid, cellSize, cellLength, rho0, radius, visc);
}

// :225-258
int PBDSolver::project(std::shared_ptr<SPHParticles>&, const std::shared_ptr<SPHParticles>&, const DArray<int>&,
                       const DArray<int>&, float rho0, int3, float3 spaceSize, float, float, int maxIter_) {
    const float sp[3] = {spaceSize.x, spaceSize.y, spaceSize.z};
    auto iter = 0;
    while (iter < maxIter_) {
        check(sphk_pbd_density_lambda(current_.ctx, &current_.abi, bufferFloat.addr(), rho0, relaxation),
              "sphk_pbd_density_lambda");
        produced(2, bufferFloat.addr(), 1);
        react(reactCoef_);      // before the positions move: the pairs of this correction
        check(sphk_pbd_delta_pos_apply(current_.ctx, &current_.abi, bufferFloat.addr(),
                                       reinterpret_cast<float*>(bufferFloat3.addr()), rho0, sp),
              "sphk_pbd_delta_pos_apply");
        produced(4, current_.abi.fluid.pos, 3);
        ++iter;
    }
    return iter;
}

// ================================================================================================
// SPHSystem (SPHSystem.cu)
// ================================================================================================
SPHSystem::SPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
                     std::shared_ptr<BaseSolver>& solver, const float3 spaceSize, const float sphCellLength,
                     const float sphSmoothingRadius, const float dt, const float sphM0, const float sphRho0,
                     const float sphRhoBoundary, const float sphStiff, const float sphVisc,
                     const float sphSurfaceTensionIntensity, const float sphAirPressure, const float3 sphG,
                     const int3 cellSize)
    : SPHSystem(fluidParticles, boundaryParticles, solver, spaceSize, sphCellLength, sphSmoothingRadius, dt, sphM0, sphRho0,
                sphRhoBoundary, sphStiff, sphVisc, sphSurfaceTensionIntensity, sphAirPressure, sphG, cellSize, {}) {}

SPHSystem::SPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
                     std::shared_ptr<BaseSolver>& solver, const float3 spaceSize, const float sphCellLength,
                     const float sphSmoothingRadius, const float dt, const float sphM0, const float sphRho0,
                     const float sphRhoBoundary, const float sphStiff, const float sphVisc,
                     const float sphSurfaceTensionIntensity, const float sphAirPressure, const float3 sphG,
                     const int3 cellSize, const std::vector<sphb200::KinematicBody>& bodies)
    : SPHSystem(fluidParticles, boundaryParticles, solver, spaceSize, sphCellLength, sphSmoothingRadius, dt, sphM0, sphRho0,
                sphRhoBoundary, sphStiff, sphVisc, sphSurfaceTensionIntensity, sphAirPressure, sphG, cellSize, bodies, {}) {}

// the caller's static boundary set followed by the bodies' particles (placed on the host here only to give the arrays a
// value: the first boundary search places them on the device)
static std::shared_ptr<SPHParticles> withBodies(std::shared_ptr<SPHParticles>&& boundary,
                                                const std::vector<sphb200::KinematicBody>& bodies) {
    if (bodies.empty()) return std::move(boundary);
    std::vector<float3> all(boundary->size());
    CUDA_CALL(cudaMemcpy(all.data(), boundary->getPosPtr(), sizeof(float3) * all.size(), cudaMemcpyDeviceToHost));
    for (const auto& b : bodies)
        for (const float3& r : b.points) all.push_back(make_float3(b.position.x + r.x, b.position.y + r.y, b.position.z + r.z));
    boundary.reset();
    return std::make_shared<SPHParticles>(all);
}

SPHSystem::SPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
                     std::shared_ptr<BaseSolver>& solver, const float3 spaceSize, const float sphCellLength,
                     const float sphSmoothingRadius, const float dt, const float sphM0, const float sphRho0,
                     const float sphRhoBoundary, const float sphStiff, const float sphVisc,
                     const float sphSurfaceTensionIntensity, const float sphAirPressure, const float3 sphG,
                     const int3 cellSize, const std::vector<sphb200::KinematicBody>& bodies,
                     const sphb200::OpenBoundaries& open)
    // the caller's three shared_ptrs are moved from, as in the reference (SPHSystem.cu:50-51)
    : _fluids(std::move(fluidParticles)), _boundaries(withBodies(std::move(boundaryParticles), bodies)), _solver(std::move(solver)),
      cellStartFluid(cellSize.x * cellSize.y * cellSize.z + 1), cellStartBoundary(cellSize.x * cellSize.y * cellSize.z + 1),
      _spaceSize(spaceSize), _sphSmoothingRadius(sphSmoothingRadius), _sphCellLength(sphCellLength), _dt(dt),
      _sphRho0(sphRho0), _sphRhoBoundary(sphRhoBoundary), _sphStiff(sphStiff), _sphG(sphG), _sphVisc(sphVisc),
      _sphSurfaceTensionIntensity(sphSurfaceTensionIntensity), _sphAirPressure(sphAirPressure), _cellSize(cellSize) {
    _engine = std::make_shared<sphb200::Engine>(static_cast<int>(_fluids->capacity()), boundarySize(), cellSize, sphCellLength);
    _fluids->bindEngine(_engine);
    _boundaries->bindEngine(_engine);
    CUDA_CALL(cudaEventCreate(&_evStart));
    CUDA_CALL(cudaEventCreate(&_evStop));
    if (const char* g = std::getenv("SPHK_STEP_GRAPH")) _graphEnabled = g[0] != '0';
    _stepDt = _lastDt = dt;
    if (!_engine->ok()) return;
    _sphM0 = sphM0;
    if (!open.emitters.empty() || !open.sinks.empty()) {
        if (const char* why = openRefusal(open)) {
            printf("SPHSystem: open boundaries refused (%s); the system is closed\n", why);
        } else {
            for (const auto& e : open.emitters) {
                sphk_emitter k;
                k.origin[0] = e.origin.x; k.origin[1] = e.origin.y; k.origin[2] = e.origin.z;
                k.direction[0] = e.direction.x; k.direction[1] = e.direction.y; k.direction[2] = e.direction.z;
                k.speed = e.speed; k.spacing = e.spacing; k.width = e.width; k.height = e.height;
                _emitters.push_back(k);
            }
            _emitterCarry.assign(_emitters.size(), 0.0);
            for (const auto& b : open.sinks) _sinkBoxes.insert(_sinkBoxes.end(), {b.lo.x, b.lo.y, b.lo.z, b.hi.x, b.hi.y, b.hi.z});
            _open = true;
        }
    }
    if (!bodies.empty()) {
        const int nStatic = boundarySize() - static_cast<int>(std::accumulate(
            bodies.begin(), bodies.end(), size_t(0), [](size_t a, const sphb200::KinematicBody& b) { return a + b.points.size(); }));
        std::vector<int> begin{nStatic};
        std::vector<float> local, pose, motion;
        for (const auto& b : bodies) {
            begin.push_back(begin.back() + static_cast<int>(b.points.size()));
            for (const float3& r : b.points) local.insert(local.end(), {r.x, r.y, r.z});
            pose.insert(pose.end(), {b.position.x, b.position.y, b.position.z, b.orientation.x, b.orientation.y, b.orientation.z,
                                     b.orientation.w});
            motion.insert(motion.end(), {b.linearVelocity.x, b.linearVelocity.y, b.linearVelocity.z, b.angularVelocity.x,
                                         b.angularVelocity.y, b.angularVelocity.z});
        }
        std::vector<float> mi;
        for (const auto& b : bodies) mi.insert(mi.end(), {b.mass, b.inertia.x, b.inertia.y, b.inertia.z});
        _bodiesHash = stateHash(local.data(), 4ull * local.size()) * 31u + stateHash(mi.data(), 4ull * mi.size()) +
                      static_cast<unsigned long long>(nStatic);
        const sphk_particles bp = _boundaries->abi();
        const int rc = sphk_bodies_init(_engine->ctx(), &bp, nStatic, static_cast<int>(bodies.size()), begin.data(),
                                        local.data(), pose.data(), motion.data());
        check(rc, "sphk_bodies_init");
        if (rc == 0) { _bodyMotion = motion; _engine->bodies = static_cast<int>(bodies.size()); }
        const bool dynamic = std::any_of(bodies.begin(), bodies.end(), [](const sphb200::KinematicBody& b) { return b.mass > 0.0f; });
        if (rc == 0 && dynamic) {
            const float sp[3] = {spaceSize.x, spaceSize.y, spaceSize.z};
            const int rd = sphk_bodies_set_dynamics(_engine->ctx(), mi.data(), sp);
            check(rd, "sphk_bodies_set_dynamics");
            _bodiesDynamic = _engine->bodiesDynamic = rd == 0;
        }
    }
    // SPHSystem.cu:68-76 (with bodies the boundary search also places them at their initial pose)
    neighborSearch(_boundaries, cellStartBoundary);
    computeBoundaryMass();
    check(sphk_fill(_engine->ctx(), _fluids->getMassPtr(), fluidSize(), sphM0), "sphk_fill");
    neighborSearch(_fluids, cellStartFluid);
    step();
}

SPHSystem::~SPHSystem() noexcept {
    if (_engine && _engine->ok()) sphk_synchronize(_engine->ctx());
    if (_graphExec) cudaGraphExecDestroy(_graphExec);
    sphk_probe_series_destroy(_probeSeries);
    if (_evStart) cudaEventDestroy(_evStart);
    if (_evStop) cudaEventDestroy(_evStop);
}

// SPHSystem.cu:107-112
void SPHSystem::computeBoundaryMass() {
    const sphk_particles b = _boundaries->abi();
    check(sphk_boundary_mass(_engine->ctx(), &b, cellStartBoundary.addr(), _sphRhoBoundary, _sphSmoothingRadius),
          "sphk_boundary_mass");
}

// SPHSystem.cu:114-127
void SPHSystem::neighborSearch(const std::shared_ptr<SPHParticles>& particles, DArray<int>& cellStart) {
    const sphk_particles p = particles->abi();
    const int which = (particles.get() == _boundaries.get()) ? 1 : 0;
    check(sphk_neighbor_search(_engine->ctx(), which, &p, cellStart.addr()), "sphk_neighbor_search");
    // the fluid search re-packs the records from the API arrays: edits made behind the engine's back
    // (Particles::advect, raw pointer writes) are absorbed here, no separate sphk_refresh is needed
    if (which == 0) _engine->shadowsStale = false;
}

// With open boundaries (DESIGN.md section 2.6): sinks and emitters, the bodies, the search over n + e slots, then the live count
// L = n + e - removed (the wait for the sinks' count overlaps the search).
void SPHSystem::searchForStep() {
    const int n = fluidSize();
    const int e = _open ? openEmit(n) : 0;
    if (!_bodyMotion.empty()) {
        const sphk_particles b = _boundaries->abi();
        check(sphk_bodies_step(_engine->ctx(), &b, cellStartBoundary.addr(), _stepDt), "sphk_bodies_step");
    }
    if (!_open) { neighborSearch(_fluids, cellStartFluid); return; }
    _fluids->setActiveCount(n + e);
    if (n + e == 0) return;
    neighborSearch(_fluids, cellStartFluid);
    int removed = 0;
    if (!_sinkBoxes.empty()) check(sphk_sinks_removed(_engine->ctx(), &removed), "sphk_sinks_removed");
    const int live = n + e - removed;
    check(sphk_fluid_set_count(_engine->ctx(), cellStartFluid.addr(), live), "sphk_fluid_set_count");
    _fluids->setActiveCount(live);
    _openStats.removed += removed;
}

// the sinks over the n live slots, then every emitter's scheduled layers into the slots after them
int SPHSystem::openEmit(int n) {
    sphk_ctx* ctx = _engine->ctx();
    const sphk_particles f = _fluids->abi();
    if (!_sinkBoxes.empty())
        check(sphk_sinks_apply(ctx, &f, _sinkBoxes.data(), static_cast<int>(_sinkBoxes.size() / 6)), "sphk_sinks_apply");
    int width = 0;
    auto* solver = dynamic_cast<BasicSPHSolver*>(_solver.get());
    float* history = solver->historyArray(width);
    const float historyDt = solver->historyTimeStep(_stepDt);
    const int kind = width == 1 ? 1 : width == 3 ? 2 : 0;
    const int cap = static_cast<int>(_fluids->capacity());
    int e = 0;
    for (size_t k = 0; k < _emitters.size(); ++k) {
        const sphk_emitter& em = _emitters[k];
        const int per = em.width * em.height;
        const int fit = std::min((cap - n - e) / per, 65536);
        if (static_cast<int>(_layerOffsets.size()) < fit) _layerOffsets.resize(static_cast<size_t>(fit));
        int scheduled = 0;
        const int rc = sphk_emitter_advance(&em, &_emitterCarry[k], _stepDt, fit, _layerOffsets.data(), &scheduled);
        check(rc, "sphk_emitter_advance");
        if (rc != 0) continue;
        const int layers = std::min(scheduled, fit);
        _openStats.refused += static_cast<long long>(scheduled - layers) * per;
        if (layers == 0) continue;
        check(sphk_emit(ctx, &f, n + e, &em, layers, _layerOffsets.data(), _sphM0, historyDt, kind ? history : nullptr, kind), "sphk_emit");
        if (solver->thermalOn()) {          // the emitter's temperature (default Tref) into its new slots
            const sphb200::Thermal& th = solver->thermal();
            check(sphk_fill(ctx, solver->temperatureField().addr(n + e), layers * per, k < th.emitterT.size() ? th.emitterT[k] : th.Tref),
                  "sphk_fill");
        }
        e += layers * per;
        _openStats.emitted += static_cast<long long>(layers) * per;
    }
    return e;
}

// why the constructor refuses the open boundaries (nullptr: accepted)
const char* SPHSystem::openRefusal(const sphb200::OpenBoundaries& open) const {
    const auto* basic = dynamic_cast<const BasicSPHSolver*>(_solver.get());
    if (!basic) return "the solver is not a BasicSPHSolver, so its history array is unknown";
    if (basic->capacity() < static_cast<int>(_fluids->capacity())) return "the solver's buffers are smaller than the fluid's capacity";
    if (open.emitters.size() > SPHK_MAX_EMITTERS || open.sinks.size() > SPHK_MAX_SINKS) return "more than 16 emitters or sinks";
    const float clamp[3] = {0.99f * _spaceSize.x, 0.99f * _spaceSize.y, 0.99f * _spaceSize.z};
    for (const auto& s : open.sinks) {
        const float b[6] = {s.lo.x, s.lo.y, s.lo.z, s.hi.x, s.hi.y, s.hi.z};
        for (int a = 0; a < 3; ++a)
            if (!std::isfinite(b[a]) || !std::isfinite(b[3 + a]) || !(b[a] < b[3 + a])) return "a sink needs finite lo < hi on every axis";
    }
    for (const auto& e : open.emitters) {
        sphk_emitter k;
        k.origin[0] = e.origin.x; k.origin[1] = e.origin.y; k.origin[2] = e.origin.z;
        k.direction[0] = e.direction.x; k.direction[1] = e.direction.y; k.direction[2] = e.direction.z;
        k.speed = e.speed; k.spacing = e.spacing; k.width = e.width; k.height = e.height;
        float ax[9];
        if (sphk_emitter_axes(&k, ax) != 0) return "an emitter needs finite values, |direction| > 0, speed > 0, spacing > 0, width and height >= 1";
        // the corners of the layer, and of the layer advanced by speed * dt, in the kernel's float operations
        for (int c = 0; c < 8; ++c) {
            const float ta = ((c & 1) ? 0.5f : -0.5f) * static_cast<float>(e.width - 1) * e.spacing;
            const float tb = ((c & 2) ? 0.5f : -0.5f) * static_cast<float>(e.height - 1) * e.spacing;
            const float delta = (c & 4) ? e.speed * _dt : 0.0f;
            for (int a = 0; a < 3; ++a) {
                const float x = k.origin[a] + ta * ax[3 + a] + tb * ax[6 + a] + delta * ax[a];
                if (!(x >= 0.0f && x <= clamp[a])) return "an emitter's layer reaches outside the clamp box [0, 0.99 spaceSize]";
            }
        }
    }
    return nullptr;
}

int SPHSystem::openBoundaryCheck() const {
    int bits = 0;
    if (_engine->ok()) check(sphk_open_check(_engine->ctx(), &bits), "sphk_open_check");
    return bits;
}

// ---- tank motion (DESIGN.md section 2.15) ----
static bool tankMotionAbi(const sphb200::TankMotion& m, sphk_tank_motion& a) {
    std::memset(&a, 0, sizeof(a));
    if (m.harmonics.size() > SPHK_TANK_HARMONICS) return false;
    a.axis[0] = m.axis.x; a.axis[1] = m.axis.y; a.axis[2] = m.axis.z;
    a.pivot[0] = m.pivot.x; a.pivot[1] = m.pivot.y; a.pivot[2] = m.pivot.z;
    a.roll_amplitude = m.rollAmplitude; a.roll_omega = m.rollOmega; a.roll_phase = m.rollPhase; a.spin = m.spin;
    a.accel[0] = m.accel.x; a.accel[1] = m.accel.y; a.accel[2] = m.accel.z;
    a.n_harmonics = static_cast<int>(m.harmonics.size());
    for (size_t k = 0; k < m.harmonics.size(); ++k) {
        const auto& h = m.harmonics[k];
        a.harmonic_amplitude[k][0] = h.amplitude.x; a.harmonic_amplitude[k][1] = h.amplitude.y; a.harmonic_amplitude[k][2] = h.amplitude.z;
        a.harmonic_omega[k] = h.omega; a.harmonic_phase[k] = h.phase;
    }
    a.ramp = m.ramp;
    return true;
}

double SPHSystem::ruleGravity() const {
    const float g[3] = {_sphG.x, _sphG.y, _sphG.z};
    if (_tankOn) {
        const float sp[3] = {_spaceSize.x, _spaceSize.y, _spaceSize.z};
        double b = 0.0;
        check(sphk_tank_accel_bound(&_tankAbi, g, sp, &b), "sphk_tank_accel_bound");
        return b;
    }
    return std::sqrt(double(g[0]) * g[0] + double(g[1]) * g[1] + double(g[2]) * g[2]);
}

bool SPHSystem::setTankMotion(const sphb200::TankMotion& m) {
    auto* solver = dynamic_cast<BasicSPHSolver*>(_solver.get());
    if (!_engine->ok() || !solver) {
        printf("setTankMotion: needs a working engine and one of the shipped solvers; the setting is kept\n");
        return false;
    }
    sphk_tank_motion a;
    const float g[3] = {_sphG.x, _sphG.y, _sphG.z};
    float probe[SPHK_TANK_STATE];
    if (!tankMotionAbi(m, a) || sphk_tank_eval(&a, g, 0.0, probe) != 0) {
        printf("setTankMotion: need finite values, a non-zero axis, rollOmega, harmonic omegas and ramp >= 0 and at most %d harmonics; "
               "the setting is kept\n", SPHK_TANK_HARMONICS);
        return false;
    }
    if (solver->thermalOn()) {
        printf("setTankMotion: not together with heat transfer (the Boussinesq buoyancy acts along the constant G); the setting is "
               "kept\n");
        return false;
    }
    const bool rotates = a.roll_amplitude != 0.0f || a.spin != 0.0f;
    if (rotates && _bodiesDynamic) {
        printf("setTankMotion: a rotating tank is not supported with dynamic bodies; the setting is kept\n");
        return false;
    }
    check(sphk_tank_set(_engine->ctx(), &a, g), "sphk_tank_set");
    // the motion is a function of the simulated time: the frame time starts where the system is
    check(sphk_tank_set_time(_engine->ctx(), _simTime), "sphk_tank_set_time");
    dropStepGraph();                        // the graph holds the motion of its capture
    _tankOn = true; _tankAbi = a;
    solver->setTankForce(true);
    if (_adaptive) _rule.gravity = ruleGravity();
    return true;
}

void SPHSystem::clearTankMotion() {
    if (!_tankOn) return;
    check(sphk_tank_set(_engine->ctx(), nullptr, nullptr), "sphk_tank_set");
    dropStepGraph();
    _tankOn = false;
    if (auto* solver = dynamic_cast<BasicSPHSolver*>(_solver.get())) solver->setTankForce(false);
    if (_adaptive) _rule.gravity = ruleGravity();
}

sphb200::TankState SPHSystem::tankState() const {
    sphb200::TankState s;
    s.t = _simTime;
    const float g[3] = {_sphG.x, _sphG.y, _sphG.z};
    float e[SPHK_TANK_STATE] = {0, 0, 0, g[0], g[1], g[2], 0, 0, 0};
    if (_tankOn) check(sphk_tank_eval(&_tankAbi, g, _simTime, e), "sphk_tank_eval");
    s.theta = e[0]; s.thetaDot = e[1]; s.thetaDDot = e[2];
    s.gravity = make_float3(e[3], e[4], e[5]);
    s.accel = make_float3(e[6], e[7], e[8]);
    return s;
}

// the end of a step with dynamic bodies (after the solver's last reaction, inside a captured step graph)
void SPHSystem::integrateBodies() {
    if (!_bodiesDynamic) return;
    const float g[3] = {_sphG.x, _sphG.y, _sphG.z};
    check(sphk_bodies_integrate(_engine->ctx(), _stepDt, g), "sphk_bodies_integrate");
}

void SPHSystem::setBodyMotion(int body, float3 linearVelocity, float3 angularVelocity) {
    if (body < 0 || body >= bodyCount()) { printf("setBodyMotion: no body %d (the system has %d)\n", body, bodyCount()); return; }
    if (!_engine->ok()) return;
    const float m[6] = {linearVelocity.x, linearVelocity.y, linearVelocity.z, angularVelocity.x, angularVelocity.y, angularVelocity.z};
    // this body only: the host copy of a dynamic body's motion is stale, the device holds the integrated one
    const int rc = sphk_bodies_set_body_motion(_engine->ctx(), body, m);   // refuses non-finite values: the motion is kept
    check(rc, "sphk_bodies_set_body_motion");
    if (rc == 0) std::copy(m, m + 6, _bodyMotion.begin() + 6 * body);
    refreshSpeedBound();                    // the next step's dt must see the new motion (enqueued after its copy)
}

void SPHSystem::getBodyMotion(int body, float3& linearVelocity, float3& angularVelocity) const {
    if (body < 0 || body >= bodyCount()) { printf("getBodyMotion: no body %d (the system has %d)\n", body, bodyCount()); return; }
    std::vector<float> motion(6 * static_cast<size_t>(bodyCount()));
    if (!_engine->ok()) return;
    check(sphk_bodies_get_motion(_engine->ctx(), motion.data()), "sphk_bodies_get_motion");
    const float* M = motion.data() + 6 * body;
    linearVelocity = make_float3(M[0], M[1], M[2]);
    angularVelocity = make_float3(M[3], M[4], M[5]);
}

void SPHSystem::getBodyImpulse(int body, float3& linearImpulse, float3& angularImpulse) const {
    if (body < 0 || body >= bodyCount()) { printf("getBodyImpulse: no body %d (the system has %d)\n", body, bodyCount()); return; }
    std::vector<float> imp(6 * static_cast<size_t>(bodyCount()), 0.0f);
    if (!_engine->ok()) return;
    if (_bodiesDynamic) check(sphk_bodies_get_impulse(_engine->ctx(), imp.data()), "sphk_bodies_get_impulse");
    const float* I = imp.data() + 6 * body;
    linearImpulse = make_float3(I[0], I[1], I[2]);
    angularImpulse = make_float3(I[3], I[4], I[5]);
}

void SPHSystem::getBodyPose(int body, float3& position, float4& orientation) const {
    if (body < 0 || body >= bodyCount()) { printf("getBodyPose: no body %d (the system has %d)\n", body, bodyCount()); return; }
    std::vector<float> pose(7 * static_cast<size_t>(bodyCount()));
    if (!_engine->ok()) return;
    check(sphk_bodies_get_pose(_engine->ctx(), pose.data()), "sphk_bodies_get_pose");
    const float* P = pose.data() + 7 * body;
    position = make_float3(P[0], P[1], P[2]);
    orientation = make_float4(P[3], P[4], P[5], P[6]);
}

// SPHSystem.cu:129-158
bool SPHSystem::solverIsGraphSafe() const {
    const auto* known = dynamic_cast<const BasicSPHSolver*>(_solver.get());   // unknown BaseSolver subclasses: never
    return known && known->stepIsGraphSafe();
}

unsigned int SPHSystem::solverConfigEpoch() const {
    const auto* known = dynamic_cast<const BasicSPHSolver*>(_solver.get());
    return known ? known->configEpoch() : 0u;
}

void SPHSystem::dropStepGraph() {
    if (!_graphExec) return;
    sphk_synchronize(_engine->ctx());
    cudaGraphExecDestroy(_graphExec);
    _graphExec = nullptr;
}

void SPHSystem::setStepGraph(bool on) {
    _graphEnabled = on;
    if (!on) dropStepGraph();
}

// SPHSystem.cu:129-158.  Small scenes are launch-bound (~45 kernels of a few microseconds per DFSPH step): once
// two plain steps have run (all lazy allocations done), a fixed-iteration step is captured into a CUDA graph and
// replayed -- same kernels, same order, same arguments (all scene parameters are const members).
float SPHSystem::step() {
    if (!_engine->ok()) return 0.0f;
    bool frameEnd = false;
    _stepDt = _adaptive ? chooseTimeStep(0.0, frameEnd) : _dt;
    return runStep();
}

// ---- CFL-adaptive time stepping (DESIGN.md section 2.8) ----
bool SPHSystem::setAdaptiveTimeStep(float C, float dtMin, float dtMax) {
    sphk_time_step_rule r;
    r.cfl = C;
    r.dt_max = dtMax > 0.0f ? dtMax : _dt;
    r.dt_min = dtMin > 0.0f ? dtMin : static_cast<float>(r.dt_max) / 64.0f;
    r.radius = _sphSmoothingRadius;
    r.gravity = ruleGravity();
    float dt = 0.0f;
    int flags = 0;
    // the library's rule validates its own parameters
    if (dtMin < 0.0f || dtMax < 0.0f || sphk_time_step(&r, 0.0, 0.0, 0.0, &dt, &flags) != 0) {
        printf("setAdaptiveTimeStep: need C > 0, dtMin >= 0 and dtMax >= 0 (finite; 0 = the default) with dtMin <= dtMax (got %g, %g, "
               "%g); the setting is kept\n", C, dtMin, dtMax);
        return false;
    }
    // the constructor checked that every emitted layer, advanced by speed * dt, stays inside the clamp box: a longer step could
    // emit past it
    if (!_emitters.empty() && r.dt_max > _dt) {
        printf("setAdaptiveTimeStep: dtMax %g is above the constructor's dt %g, for which the emitters were checked; the setting is "
               "kept\n", dtMax, _dt);
        return false;
    }
    dropStepGraph();
    _rule = r;
    _adaptive = true;
    if (_engine->ok()) measureSpeed();       // the bound of the current state, for the first adaptive step
    return true;
}

void SPHSystem::refreshSpeedBound() {
    if (_adaptive && _engine->ok()) measureSpeed();
}

void SPHSystem::disableAdaptiveTimeStep() {
    if (!_adaptive) return;
    _adaptive = false;
    _plainSteps = 0;       // a PBD step still derives its velocities over the last adaptive dt: capture after two fixed steps
}

int SPHSystem::advance(double frameSeconds) {
    if (!_adaptive || !(frameSeconds > 0.0) || !std::isfinite(frameSeconds)) {
        printf("SPHSystem::advance: needs an adaptive system (setAdaptiveTimeStep) and a finite frame > 0 (got %g)\n", frameSeconds);
        return 0;
    }
    if (!_engine->ok()) return 0;
    double elapsed = 0.0;
    int steps = 0;
    bool frameEnd = false;
    float minDt = std::numeric_limits<float>::max();
    while (!frameEnd) {
        _stepDt = chooseTimeStep(frameSeconds - elapsed, frameEnd);
        runStep();
        elapsed += _stepDt;
        minDt = std::min(minDt, _stepDt);
        ++steps;
    }
    _adaptiveStats.frameMinDt = minDt;
    return steps;
}

void SPHSystem::measureSpeed() {
    const sphk_particles f = _fluids->abi();
    check(sphk_step_speed(_engine->ctx(), &f, _bodyMotion.empty() ? 0 : 1), "sphk_step_speed");
}

float SPHSystem::chooseTimeStep(double remaining, bool& frameEnd) {
    float v[2] = {0.0f, 0.0f};
    int nonFinite = 0;
    check(sphk_step_speed_result(_engine->ctx(), v, &nonFinite), "sphk_step_speed_result");
    float vmax = v[0];
    int source = 0;
    if (v[1] > vmax) { vmax = v[1]; source = 1; }
    for (const auto& e : _emitters)
        if (e.speed > vmax) { vmax = e.speed; source = 2; }
    float dt = _rule.dt_min;
    int flags = SPHK_DT_NONFINITE;
    const int rc = sphk_time_step(&_rule, vmax, _lastDt, remaining, &dt, &flags);
    check(rc, "sphk_time_step");
    _adaptiveStats.speed = vmax;
    _adaptiveStats.source = source;
    if (flags & SPHK_DT_MIN_CLAMP) ++_adaptiveStats.minClamps;
    if ((flags & SPHK_DT_NONFINITE) || nonFinite > 0) ++_adaptiveStats.nonFiniteSteps;
    frameEnd = rc != 0 || (flags & SPHK_DT_FRAME_END) != 0;
    return dt;
}

float SPHSystem::runStep() {
    cudaStream_t st = _engine->stream();
    sphk_ctx* ctx = _engine->ctx();
    CUDA_CALL(cudaEventRecord(_evStart, st));
    // a captured step replays a fixed kernel sequence: drop it when the solver's settings changed or it stopped being
    // replayable.  (Particles moved behind the engine's back need nothing special: the replayed step begins with the
    // fluid neighbour search, which re-packs the records from the API arrays.)
    if (_graphExec && (_graphConfigEpoch != solverConfigEpoch() || !solverIsGraphSafe())) dropStepGraph();
    _probeRecorded = false;
    if (_graphExec) {
        _engine->shadowsStale = false;
        _probeRecorded = _probeSeries != nullptr;     // (a series set or cleared drops the graph: it was captured with this one)
        CUDA_CALL(cudaGraphLaunch(_graphExec, st));
        sphk_add_launches(ctx, _graphLaunches);
        check(sphk_synchronize(ctx), "step");
    } else {
        const bool capture = _graphEnabled && !_open && !_adaptive && _plainSteps >= 2 && solverIsGraphSafe();
        const long long launches0 = sphk_launch_count(ctx);
        bool captured = false;
        if (capture) captured = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
        bool ok = false;
        try {
            searchForStep();
            if (fluidSize() > 0)        // (an open system can run empty)
                _solver->step(_fluids, _boundaries, cellStartFluid, cellStartBoundary, _spaceSize, _cellSize, _sphCellLength,
                              _sphSmoothingRadius, _stepDt, _sphRho0, _sphRhoBoundary, _sphStiff, _sphVisc, _sphG,
                              _sphSurfaceTensionIntensity, _sphAirPressure);
            integrateBodies();
            recordProbes();
            if (_adaptive) measureSpeed();      // after the step's last velocity write; read before the next step
            ok = true;
        } catch (const char* s) {
            std::cout << s << "\n";
        } catch (...) {
            std::cout << "Unknown Exception at " << __FILE__ << ": line " << __LINE__ << "\n";
        }
        if (captured) {
            cudaGraph_t graph = nullptr;
            if (cudaStreamEndCapture(st, &graph) == cudaSuccess && graph && ok &&
                cudaGraphInstantiate(&_graphExec, graph, 0) == cudaSuccess) {
                _graphLaunches = sphk_launch_count(ctx) - launches0;
                _graphConfigEpoch = solverConfigEpoch();
                CUDA_CALL(cudaGraphLaunch(_graphExec, st));     // the captured step has not run yet: run it now
            } else {
                cudaGetLastError();
                _graphExec = nullptr;
                _graphEnabled = false;                          // capture refused (e.g. a library call): stay on plain launches
                printf("SPHSystem: step graph capture failed, continuing with plain launches\n");
                searchForStep();
                try {
                    _solver->step(_fluids, _boundaries, cellStartFluid, cellStartBoundary, _spaceSize, _cellSize,
                                  _sphCellLength, _sphSmoothingRadius, _stepDt, _sphRho0, _sphRhoBoundary, _sphStiff, _sphVisc,
                                  _sphG, _sphSurfaceTensionIntensity, _sphAirPressure);
                    integrateBodies();
                    recordProbes();
                } catch (const char* s) {
                    std::cout << s << "\n";
                } catch (...) {
                    std::cout << "Unknown Exception at " << __FILE__ << ": line " << __LINE__ << "\n";
                }
            }
            if (graph) cudaGraphDestroy(graph);
        }
        if (ok) ++_plainSteps;
        check(sphk_synchronize(ctx), "step");
    }
    _lastDt = _stepDt;
    _simTime += _stepDt;
    _restored = false;
    if (_probeRecorded) {                        // the row recordProbes() enqueued: its step and time
        const size_t slot = static_cast<size_t>(_probeRows % _probes.capacity);
        _probeSteps[slot] = _steps;
        _probeTimes[slot] = _simTime;
        ++_probeRows;
    }
    ++_steps;
    float milliseconds = 0.0f;
    CUDA_CALL(cudaEventRecord(_evStop, st));
    CUDA_CALL(cudaEventSynchronize(_evStop));
    CUDA_CALL(cudaEventElapsedTime(&milliseconds, _evStart, _evStop));
    return milliseconds;
}

// ---- probes and water-level gauges (DESIGN.md section 2.13) ----
sphk_scene SPHSystem::probeScene() const {
    sphk_scene s{};
    s.fluid = _fluids->abi();
    s.boundary = _boundaries->abi();
    s.cell_start_fluid = cellStartFluid.addr();
    s.cell_start_boundary = cellStartBoundary.addr();
    s.radius = _sphSmoothingRadius;
    return s;
}

// the pressure a WCSPH step computed (DFSPH and PBD keep none), and the temperatures while heat transfer is on
void SPHSystem::probeSources(const float*& pressure, const float*& temperature) const {
    auto* basic = dynamic_cast<BasicSPHSolver*>(_solver.get());
    pressure = basic && typeid(*basic) == typeid(BasicSPHSolver) ? _fluids->getPressurePtr() : nullptr;
    temperature = basic && basic->thermalOn() ? basic->temperatureField().addr() : nullptr;
}

void SPHSystem::recordProbes() {
    if (!_probeSeries || fluidSize() == 0) return;     // (an open system that runs empty records no row)
    const sphk_scene s = probeScene();
    const float *p = nullptr, *t = nullptr;
    probeSources(p, t);
    const int rc = sphk_probes_record(_engine->ctx(), &s, _probeSeries, p, t);
    check(rc, "sphk_probes_record");
    _probeRecorded = rc == 0;
}

bool SPHSystem::setProbes(const sphb200::Probes& probes) {
    std::vector<float> pts;
    for (const float3& q : probes.points) pts.insert(pts.end(), {q.x, q.y, q.z});
    std::vector<sphk_gauge> gs;
    for (const auto& g : probes.gauges) gs.push_back(sphk_gauge{{g.a.x, g.a.y, g.a.z}, {g.b.x, g.b.y, g.b.z}, g.samples});
    if (probes.points.size() > SPHK_PROBE_LIMIT || probes.gauges.size() > SPHK_GAUGE_LIMIT) {
        printf("setProbes: at most %d probes and %d gauges (got %zu, %zu); the setting is kept\n", SPHK_PROBE_LIMIT, SPHK_GAUGE_LIMIT,
               probes.points.size(), probes.gauges.size());
        return false;
    }
    if (!_engine->ok()) return false;
    sphk_probe_series* series = nullptr;
    const int rc = sphk_probe_series_create(&series, pts.data(), static_cast<int>(probes.points.size()), gs.data(),
                                            static_cast<int>(gs.size()), probes.threshold, probes.capacity, _engine->stream());
    if (rc != 0) {
        printf("setProbes: refused (%s): need finite points, gauges with a != b and 2..%d samples, a finite threshold > 0, a capacity "
               "in [1, %d] and at least one probe or gauge; the setting is kept\n", sphk_error_string(rc), SPHK_GAUGE_MAX_SAMPLES,
               SPHK_PROBE_CAPACITY_LIMIT);
        return false;
    }
    dropStepGraph();
    sphk_probe_series_destroy(_probeSeries);
    _probeSeries = series;
    _probes = probes;
    _probeSteps.assign(static_cast<size_t>(probes.capacity), 0);
    _probeTimes.assign(static_cast<size_t>(probes.capacity), 0.0);
    _probeRows = 0;
    return true;
}

void SPHSystem::clearProbes() {
    if (!_probeSeries) return;
    dropStepGraph();
    sphk_probe_series_destroy(_probeSeries);
    _probeSeries = nullptr;
}

sphb200::ProbeSeries SPHSystem::probeSeries() const {
    sphb200::ProbeSeries out;
    if (!_probeSeries) return out;
    out.probes = static_cast<int>(_probes.points.size());
    out.gauges = static_cast<int>(_probes.gauges.size());
    const int cap = _probes.capacity;
    out.records.resize(static_cast<size_t>(cap) * out.probes * SPHK_PROBE_FIELDS);
    out.levels.resize(static_cast<size_t>(cap) * out.gauges);
    long long count = 0;
    int rows = 0;
    const int rc = sphk_probe_series_read(_probeSeries, &count, cap, out.records.data(), out.levels.data(), &rows);
    check(rc, "sphk_probe_series_read");
    if (rc != 0) rows = 0;
    if (rc == 0 && count != _probeRows) printf("probeSeries: the device recorded %lld rows, the host %lld\n", count, _probeRows);
    out.records.resize(static_cast<size_t>(rows) * out.probes * SPHK_PROBE_FIELDS);
    out.levels.resize(static_cast<size_t>(rows) * out.gauges);
    for (long long r = count - rows; r < count; ++r) {
        out.steps.push_back(_probeSteps[static_cast<size_t>(r % cap)]);
        out.times.push_back(_probeTimes[static_cast<size_t>(r % cap)]);
    }
    out.overwritten = count - rows;
    return out;
}

std::vector<float> SPHSystem::sampleProbes(const std::vector<float3>& points) const {
    std::vector<float> out;
    if (_restored) {
        printf("%s: refused until the first step after a restore (no search has run for the restored positions)\n", __func__);
        return out;
    }
    if (!_engine->ok() || points.empty() || fluidSize() == 0) return out;
    const size_t n = points.size();
    float *dp = nullptr, *dout = nullptr;
    CUDA_CALL(cudaMalloc(&dp, 12 * n));
    CUDA_CALL(cudaMalloc(&dout, 32 * n));
    CUDA_CALL(cudaMemcpyAsync(dp, points.data(), 12 * n, cudaMemcpyHostToDevice, _engine->stream()));
    const sphk_scene s = probeScene();
    const float *p = nullptr, *t = nullptr;
    probeSources(p, t);
    const int rc = sphk_probe_sample(_engine->ctx(), &s, dp, static_cast<int>(n), p, t, dout);
    check(rc, "sphk_probe_sample");
    if (rc == 0) {
        out.resize(8 * n);
        CUDA_CALL(cudaMemcpyAsync(out.data(), dout, 32 * n, cudaMemcpyDeviceToHost, _engine->stream()));
    }
    check(sphk_synchronize(_engine->ctx()), "sphk_synchronize");
    cudaFree(dp);
    cudaFree(dout);
    return out;
}

std::vector<float> SPHSystem::sampleLattice(float3 origin, float spacing, int3 dims) const {
    std::vector<float> out;
    if (_restored) {
        printf("%s: refused until the first step after a restore (no search has run for the restored positions)\n", __func__);
        return out;
    }
    if (!_engine->ok() || fluidSize() == 0) return out;
    const long long total = static_cast<long long>(dims.x) * dims.y * dims.z;
    if (dims.x < 1 || dims.y < 1 || dims.z < 1 || total > (1LL << 27)) {
        printf("sampleLattice: dims must be >= 1 with at most 2^27 points (got %d x %d x %d)\n", dims.x, dims.y, dims.z);
        return out;
    }
    float* dout = nullptr;
    CUDA_CALL(cudaMalloc(&dout, 32 * static_cast<size_t>(total)));
    const sphk_scene s = probeScene();
    const float *p = nullptr, *t = nullptr;
    probeSources(p, t);
    const float o[3] = {origin.x, origin.y, origin.z};
    const int d[3] = {dims.x, dims.y, dims.z};
    const int rc = sphk_probe_lattice(_engine->ctx(), &s, o, spacing, d, p, t, dout);
    check(rc, "sphk_probe_lattice");
    if (rc == 0) {
        out.resize(8 * static_cast<size_t>(total));
        CUDA_CALL(cudaMemcpyAsync(out.data(), dout, 32 * static_cast<size_t>(total), cudaMemcpyDeviceToHost, _engine->stream()));
    }
    check(sphk_synchronize(_engine->ctx()), "sphk_synchronize");
    cudaFree(dout);
    return out;
}

// ---- checkpoints (DESIGN.md section 2.14) ----
static sphk_state_section stateSection(const char* name, const void* p, unsigned long long bytes, unsigned int elem, bool host) {
    sphk_state_section s{};
    std::snprintf(s.name, sizeof(s.name), "%s", name);
    s.ptr = const_cast<void*>(p); s.bytes = bytes; s.elem_size = elem; s.host = host ? 1 : 0;
    return s;
}

template <typename T>
static void putBytes(std::vector<unsigned char>& v, const T& x) {
    const auto* p = reinterpret_cast<const unsigned char*>(&x);
    v.insert(v.end(), p, p + sizeof(T));
}

bool BasicSPHSolver::stateSections(std::vector<sphk_state_section>& out, int n) {
    if (typeid(*this) != typeid(BasicSPHSolver)) return false;
    commonStateSections(out, n);
    return true;
}

void BasicSPHSolver::commonStateSections(std::vector<sphk_state_section>& out, int n) {
    if (!thermalOn_) return;
    out.push_back(stateSection("solver.temperature", temperatureField().addr(), 4ull * n, 4, false));
    out.push_back(stateSection("solver.temperature_set", &temperatureSet_, sizeof(temperatureSet_), 1, true));
}

void BasicSPHSolver::stateConfig(sphk_state_config& c, std::vector<unsigned char>& settings) const {
    commonStateConfig(c, settings, "wcsph");
}

void BasicSPHSolver::commonStateConfig(sphk_state_config& c, std::vector<unsigned char>& settings, const char* name) const {
    std::snprintf(c.solver, sizeof(c.solver), "%s", name);
    if (fusedSweeps_) c.flags |= 1;
    putBytes(settings, vortEps_);
    if (implicitViscosityOn()) { putBytes(settings, implNu_); putBytes(settings, implNuB_); putBytes(settings, implTol_); putBytes(settings, implMaxIter_); }
    putBytes(settings, rheoOn_);
    if (rheoOn_) {
        putBytes(settings, static_cast<const sphk_rheology&>(rheo_));
        putBytes(settings, rheoBeta_); putBytes(settings, rheoTol_); putBytes(settings, rheoMaxIter_);
    }
    putBytes(settings, thermalOn_);
    if (thermalOn_) {
        putBytes(settings, thermalAbi_);
        for (float T : thermal_.emitterT) putBytes(settings, T);
        putBytes(settings, thermalViscOn_);
        if (thermalViscOn_) putBytes(settings, thermalVisc_);
    }
    putBytes(settings, adhesionOn_);
    if (adhesionOn_) putBytes(settings, adhesionAbi_);
}

bool DFSPHSolver::stateSections(std::vector<sphk_state_section>& out, int n) {
    commonStateSections(out, n);
    out.push_back(stateSection("solver.dfsph_warm_stiffness", denWarmStiff.addr(), 4ull * n, 4, false));
    return true;
}

void DFSPHSolver::stateConfig(sphk_state_config& c, std::vector<unsigned char>& settings) const {
    commonStateConfig(c, settings, "dfsph");
    if (deviceLoops_) c.flags |= 2;
    c.solver_args[0] = densityErrorThreshold; c.solver_args[1] = divergenceErrorThreshold; c.solver_args[2] = static_cast<float>(maxIter);
}

bool PBDSolver::stateSections(std::vector<sphk_state_section>& out, int n) {
    commonStateSections(out, n);
    out.push_back(stateSection("solver.pbd_pos_last", fluidPosLast.addr(), 12ull * n, 12, false));
    out.push_back(stateSection("solver.pbd_last_predict_dt", &lastPredictDt_, sizeof(lastPredictDt_), 4, true));
    out.push_back(stateSection("solver.pbd_pos_last_initialized", &posLastInitialized, sizeof(posLastInitialized), 1, true));
    return true;
}

void PBDSolver::stateConfig(sphk_state_config& c, std::vector<unsigned char>& settings) const {
    commonStateConfig(c, settings, "pbd");
    c.solver_args[0] = static_cast<float>(maxIter); c.solver_args[1] = xSPH_c; c.solver_args[2] = relaxation;
}

sphk_state_config SPHSystem::stateConfig() const {
    sphk_state_config c;
    std::memset(&c, 0, sizeof(c));
    c.capacity_fluid = static_cast<int>(_fluids->capacity());
    c.capacity_boundary = static_cast<int>(_boundaries->capacity());
    c.n_boundary = boundarySize();
    c.n_bodies = bodyCount();
    c.cell_size[0] = _cellSize.x; c.cell_size[1] = _cellSize.y; c.cell_size[2] = _cellSize.z;
    c.space_size[0] = _spaceSize.x; c.space_size[1] = _spaceSize.y; c.space_size[2] = _spaceSize.z;
    c.cell_length = _sphCellLength; c.radius = _sphSmoothingRadius; c.dt = _dt; c.m0 = _sphM0; c.rho0 = _sphRho0;
    c.rho_boundary = _sphRhoBoundary; c.stiff = _sphStiff; c.visc = _sphVisc; c.surface_tension = _sphSurfaceTensionIntensity;
    c.air_pressure = _sphAirPressure; c.gravity[0] = _sphG.x; c.gravity[1] = _sphG.y; c.gravity[2] = _sphG.z;
    if (_open) c.flags |= 4;
    if (_bodiesDynamic) c.flags |= 8;
    if (_adaptive) c.flags |= 16;
    c.bodies_hash = _bodiesHash;
    if (_open)
        c.open_hash = stateHash(_emitters.data(), sizeof(sphk_emitter) * _emitters.size()) * 31u +
                      stateHash(_sinkBoxes.data(), 4ull * _sinkBoxes.size()) + _emitters.size();
    std::vector<unsigned char> settings;
    if (const auto* solver = dynamic_cast<const BasicSPHSolver*>(_solver.get())) solver->stateConfig(c, settings);
    if (_adaptive) putBytes(settings, _rule);
    if (_tankOn) putBytes(settings, _tankAbi);
    c.settings_hash = stateHash(settings.data(), settings.size()) + settings.size();
    return c;
}

// every section of the file in its order: the fluid's n live particles, the boundary, the solver, the host counters, the user's bytes
// (the library appends the context's body and open-boundary state)
bool SPHSystem::stateSections(std::vector<sphk_state_section>& out, int n, StateRecord& rec, std::vector<double>& carry,
                              std::vector<float>& motion, const std::vector<unsigned char>& user) {
    const sphk_particles f = _fluids->abi(), b = _boundaries->abi();
    const unsigned long long nn = static_cast<unsigned long long>(n), nb = static_cast<unsigned long long>(boundarySize());
    out.push_back(stateSection("fluid.pos", f.pos, 12 * nn, 12, false));
    out.push_back(stateSection("fluid.vel", f.vel, 12 * nn, 12, false));
    out.push_back(stateSection("fluid.mass", f.mass, 4 * nn, 4, false));
    out.push_back(stateSection("fluid.density", f.density, 4 * nn, 4, false));
    out.push_back(stateSection("fluid.pressure", f.pressure, 4 * nn, 4, false));
    out.push_back(stateSection("fluid.particle2cell", f.particle2cell, 4 * nn, 4, false));
    out.push_back(stateSection("boundary.pos", b.pos, 12 * nb, 12, false));
    out.push_back(stateSection("boundary.mass", b.mass, 4 * nb, 4, false));
    auto* solver = dynamic_cast<BasicSPHSolver*>(_solver.get());
    if (!solver || !solver->stateSections(out, n)) return false;
    out.push_back(stateSection("system.record", &rec, sizeof(rec), 8, true));
    if (_open) out.push_back(stateSection("system.emitter_carry", carry.data(), 8ull * carry.size(), 8, true));
    if (!_bodyMotion.empty()) out.push_back(stateSection("system.body_motion", motion.data(), 4ull * motion.size(), 4, true));
    out.push_back(stateSection("user", user.data(), user.size(), 1, true));
    return true;
}

bool SPHSystem::checkpoint(const std::string& path, const std::vector<unsigned char>& user) {
    if (!_engine->ok()) return false;
    StateRecord rec;
    std::memset(&rec, 0, sizeof(rec));
    rec.steps = _steps; rec.emitted = _openStats.emitted; rec.removed = _openStats.removed; rec.refused = _openStats.refused;
    rec.minClamps = _adaptiveStats.minClamps; rec.nonFiniteSteps = _adaptiveStats.nonFiniteSteps; rec.simTime = _simTime;
    rec.lastDt = _lastDt; rec.stepDt = _stepDt; rec.speed = _adaptiveStats.speed; rec.frameMinDt = _adaptiveStats.frameMinDt;
    rec.source = _adaptiveStats.source; rec.live = fluidSize();
    std::vector<double> carry = _emitterCarry;
    std::vector<float> motion = _bodyMotion;
    std::vector<sphk_state_section> sections;
    if (!stateSections(sections, fluidSize(), rec, carry, motion, user)) {
        printf("SPHSystem::checkpoint: refused: the solver does not describe its state (only the shipped solvers do)\n");
        return false;
    }
    const sphk_state_config cfg = stateConfig();
    const int rc = sphk_checkpoint_save(_engine->ctx(), path.c_str(), &cfg, sections.data(), static_cast<int>(sections.size()));
    if (rc != 0) {
        printf("SPHSystem::checkpoint: refused (%s)\n", sphk_error_string(rc));
        return false;
    }
    return true;
}

bool SPHSystem::waitCheckpoint() {
    if (!_engine->ok()) return false;
    char msg[512];
    const int rc = sphk_checkpoint_wait(_engine->ctx(), msg, sizeof(msg));
    if (rc != 0) printf("SPHSystem::waitCheckpoint: the checkpoint failed: %s\n", msg[0] ? msg : sphk_error_string(rc));
    return rc == 0;
}

bool SPHSystem::restore(const std::string& path, std::vector<unsigned char>* user) {
    if (!_engine->ok()) return false;
    sphk_ctx* ctx = _engine->ctx();
    char msg[512] = {0};
    if (sphk_checkpoint_wait(ctx, msg, sizeof(msg)) != 0) printf("SPHSystem::restore: an earlier checkpoint failed: %s\n", msg);
    sphk_state_file* file = nullptr;
    if (sphk_state_open(path.c_str(), &file, msg, sizeof(msg)) != 0) {
        printf("SPHSystem::restore: refused: %s\n", msg);
        return false;
    }
    int n = fluidSize();
    unsigned long long posBytes = 0, userBytes = 0;
    if (sphk_state_section_bytes(file, "fluid.pos", &posBytes) != 0 || sphk_state_section_bytes(file, "user", &userBytes) != 0) {
        printf("SPHSystem::restore: refused: the file has no fluid.pos or user section\n");
        sphk_state_close(file);
        return false;
    }
    if (_open) {                           // an open system's live count is part of its state
        if (posBytes % 12 != 0 || posBytes / 12 > _fluids->capacity()) {
            printf("SPHSystem::restore: refused: section 'fluid.pos' holds %llu bytes, more than the capacity of %u particles\n", posBytes,
                   _fluids->capacity());
            sphk_state_close(file);
            return false;
        }
        n = static_cast<int>(posBytes / 12);
    }
    StateRecord rec;
    std::memset(&rec, 0, sizeof(rec));
    std::vector<double> carry(_emitterCarry.size());
    std::vector<float> motion(_bodyMotion.size());
    std::vector<unsigned char> userIn(static_cast<size_t>(userBytes));
    std::vector<sphk_state_section> sections;
    if (!stateSections(sections, n, rec, carry, motion, userIn)) {
        printf("SPHSystem::restore: refused: the solver does not describe its state (only the shipped solvers do)\n");
        sphk_state_close(file);
        return false;
    }
    const sphk_state_config cfg = stateConfig();
    const int rc = sphk_checkpoint_load(ctx, file, &cfg, sections.data(), static_cast<int>(sections.size()), msg, sizeof(msg));
    sphk_state_close(file);
    if (rc != 0) {
        printf("SPHSystem::restore: refused: %s\n", msg[0] ? msg : sphk_error_string(rc));
        return false;
    }
    // (the solver's host fields were written by the load itself)
    if (_open) _fluids->setActiveCount(n);
    _steps = rec.steps; _simTime = rec.simTime; _lastDt = rec.lastDt; _stepDt = rec.stepDt;
    _openStats.emitted = rec.emitted; _openStats.removed = rec.removed; _openStats.refused = rec.refused;
    _adaptiveStats.speed = rec.speed; _adaptiveStats.source = rec.source; _adaptiveStats.minClamps = rec.minClamps;
    _adaptiveStats.nonFiniteSteps = rec.nonFiniteSteps; _adaptiveStats.frameMinDt = rec.frameMinDt;
    _emitterCarry = carry;
    _bodyMotion = motion;
    if (user) *user = userIn;
    // the caches derived from the old state: the next step rebuilds them
    check(sphk_checkpoint_invalidate(ctx), "sphk_checkpoint_invalidate");
    dropStepGraph();
    _plainSteps = 0;
    dynamic_cast<BasicSPHSolver*>(_solver.get())->stateRestored();
    // the next adaptive dt: the speed bound of the restored state, measured again (a max over the same bits as the saved run's)
    if (_adaptive) measureSpeed();
    if (_tankOn) check(sphk_tank_set_time(ctx, _simTime), "sphk_tank_set_time");     // the frame time of the saved run
    check(sphk_synchronize(ctx), "sphk_synchronize");
    _restored = true;
    return true;
}

// vbo.cu:46-51
extern "C" void generate_dots(float3* dot, float3* color, const std::shared_ptr<SPHParticles> particles) {
    const auto& eng = particles->engine();
    if (!eng || !eng->ok()) { printf("generate_dots: particles are not bound to an engine\n"); return; }
    const sphk_particles p = particles->abi();
    check(sphk_export_dots(eng->ctx(), &p, reinterpret_cast<float*>(dot), reinterpret_cast<float*>(color)), "sphk_export_dots");
}
