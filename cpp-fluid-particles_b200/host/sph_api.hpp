// sph_api.hpp -- the reference's C++ class surface (DArray / Particles / SPHParticles / BaseSolver /
// BasicSPHSolver / DFSPHSolver / PBDSolver / SPHSystem) re-implemented as a thin HOST layer (plain
// g++, no device code) over the C-ABI of libsphk (include/sphk.h).  Same class names, constructor
// signatures, accessors and error behaviour as /root/reference/src/*.h so that the reference's call
// sites -- main.cpp:86,117 (particles), :119-130 (solvers), :131-134 (SPHSystem), :302 (step),
// vbo.cu:48 (accessors) -- compile and behave unchanged.  Everything underneath is new.
#pragma once

#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <functional>
#include <iostream>
#include <memory>
#include <type_traits>
#include <typeinfo>
#include <vector>

#include "sphk.h"

// ---- global.h:20-26 ---------------------------------------------------------------------------
constexpr int block_size = 256;
#ifndef EPSILON
#define EPSILON (1e-6f)
#endif
#ifndef PI
#define PI (3.14159265358979323846f)
#endif
#ifndef MAX_A
#define MAX_A (1000.0f)
#endif
// print-and-continue, like the reference (global.h:23,25)
#define CUDA_CALL(x)                                                                              \
    do {                                                                                          \
        const int sph_rc_ = static_cast<int>(x);                                                  \
        if (sph_rc_ != 0) printf("CUDA Error at %s:%d\t Error code = %d\n", __FILE__, __LINE__, sph_rc_); \
    } while (0)
#define CHECK_KERNEL()                                                                            \
    {                                                                                             \
        cudaError_t sph_err_ = cudaGetLastError();                                                \
        if (sph_err_) printf("CUDA Error at %s:%d:\t%s\n", __FILE__, __LINE__, cudaGetErrorString(sph_err_)); \
    }

namespace sphb200 {
// print-and-continue for C-ABI return codes (the reference never aborts on a CUDA error)
inline void check(int rc, const char* what) {
    if (rc != 0) printf("sphk error in %s: %s (%d)\n", what, sphk_error_string(rc), rc);
}

// One libsphk context + the stream all work of one SPHSystem is enqueued on.  Created by SPHSystem,
// shared with both particle sets so that solvers (which only receive particles through
// BaseSolver::step) can reach it.
class Engine {
public:
    Engine(int maxFluid, int maxBoundary, int3 cellSize, float cellLength, int3 origin = int3{0, 0, 0});
    ~Engine();
    Engine(const Engine&) = delete;
    Engine& operator=(const Engine&) = delete;
    sphk_ctx* ctx() const { return ctx_; }
    cudaStream_t stream() const { return stream_; }
    bool ok() const { return ctx_ != nullptr; }
    bool shadowsStale = false;   // set when a caller moved particles behind the engine's back
    bool bodiesDynamic = false;  // set by SPHSystem: the solvers follow every reacting sweep with sphk_bodies_react
private:
    sphk_ctx* ctx_ = nullptr;
    cudaStream_t stream_ = nullptr;
};

// addition: a rigid body (DESIGN.md sections 2.3, 2.4).  Its boundary particles are `points` in body coordinates; the
// system moves them every step.  With mass = 0 (the default) the motion is prescribed (a kinematic body).  With mass > 0
// the fluid pushes back: the body is integrated under the fluid's force and torque and gravity, and meets the walls.
// Mass units: the fluid's mass per unit volume is m0 / spacing^3 (about 9.57 in the reference's scenes), not rho0, so a
// body of relative density REL and volume V has mass = REL * m0 / spacing^3 * V.
struct KinematicBody {
    std::vector<float3> points;     // r_k, body coordinates (the principal axes of a dynamic body)
    float3 position;                // centre c, world frame (the centre of mass of a dynamic body)
    float4 orientation;             // unit quaternion q = (x, y, z, w): vector part in x, y, z, scalar part in w
    float3 linearVelocity;          // V, world frame
    float3 angularVelocity;         // Omega (rad/s), world frame, about the centre
    float mass = 0;                 // M > 0: dynamic (two-way coupled); 0: kinematic
    float3 inertia = {0, 0, 0};     // principal moments about the centre, body axes (all > 0 when mass > 0)
};

// addition: open boundaries (DESIGN.md section 2.6).  An emitter is a rectangular nozzle that adds a W x H layer of fluid
// particles, `spacing` apart, moving at speed * normalize(direction), every time the stream has advanced by one spacing; a sink
// is an axis-aligned box lo <= x < hi whose fluid particles are removed.  The fluid set keeps its capacity (SPHParticles'
// capacity constructor) and its live count changes between steps; a layer that does not fit is refused (counted, not emitted).
struct Emitter {
    float3 origin;                  // centre of the nozzle
    float3 direction;               // any length > 0
    float speed;                    // > 0
    float spacing;                  // > 0: within a layer and between layers (normally the fluid's particle spacing)
    int width = 1, height = 1;      // particles per layer along the nozzle's two in-plane axes (sphk_emitter_axes)
};
struct Sink {
    float3 lo, hi;                  // lo < hi on every axis
};
struct OpenBoundaries {
    std::vector<Emitter> emitters;  // at most SPHK_MAX_EMITTERS
    std::vector<Sink> sinks;        // at most SPHK_MAX_SINKS
};
struct OpenBoundaryStats {
    long long emitted = 0, removed = 0, refused = 0;   // cumulative particle counts
};
// addition: CFL-adaptive time stepping (DESIGN.md section 2.8)
struct AdaptiveStats {
    float speed = 0.0f;              // the speed bound v_max the last step's dt was chosen from
    int source = 0;                  // what set it: 0 = the fluid, 1 = a body, 2 = an emitter
    long long minClamps = 0;         // steps held at dt_min because C R / v_b was smaller
    long long nonFiniteSteps = 0;    // steps whose bound left out non-finite velocities, or was not finite
    float frameMinDt = 0.0f;         // the smallest dt of the last advance()
};
}  // namespace sphb200

// ---- DArray.h:21-54 ---------------------------------------------------------------------------
// RAII device array of float3 / float / int, zero-filled on construction, non-copyable.
template <typename T>
class DArray {
    static_assert(std::is_same<T, float3>::value || std::is_same<T, float>::value || std::is_same<T, int>::value,
                  "DArray must be of int, float or float3.");
public:
    explicit DArray(const unsigned int length) : count_(length), mem_(allocate(length)) { clear(); }
    DArray(const DArray&) = delete;
    DArray& operator=(const DArray&) = delete;
    ~DArray() noexcept = default;

    T* addr(const int offset = 0) const { return mem_.get() + offset; }
    unsigned int length() const { return count_; }
    void clear() { CUDA_CALL(cudaMemset(mem_.get(), 0, sizeof(T) * static_cast<size_t>(count_))); }

private:
    static std::shared_ptr<T> allocate(unsigned int length) {
        void* raw = nullptr;
        CUDA_CALL(cudaMalloc(&raw, sizeof(T) * static_cast<size_t>(length ? length : 1)));
        return std::shared_ptr<T>(static_cast<T*>(raw), [](T* p) { CUDA_CALL(cudaFree(p)); });
    }
    const unsigned int count_;
    const std::shared_ptr<T> mem_;
};

// ---- Particles.h:20-50 ------------------------------------------------------------------------
class Particles {
public:
    explicit Particles(const std::vector<float3>& p);
    // addition: capacity slots (at least p.size()), of which the first p.size() are live (size())
    Particles(const std::vector<float3>& p, unsigned int capacity);
    Particles(const Particles&) = delete;
    Particles& operator=(const Particles&) = delete;
    virtual ~Particles() noexcept {}

    // (addition: a slab rank keeps capacity-sized arrays of which the first activeCount_ entries are live)
    unsigned int size() const { return activeCount_ >= 0 ? static_cast<unsigned int>(activeCount_) : pos.length(); }
    unsigned int capacity() const { return pos.length(); }
    void setActiveCount(int n) { activeCount_ = n; }
    float3* getPosPtr() const { return pos.addr(); }
    float3* getVelPtr() const { return vel.addr(); }
    const DArray<float3>& getPos() const { return pos; }
    void advect(float dt);   // pos += dt * vel (Particles.cu:28-36)

    // -- additions (not in the reference): engine binding, set by SPHSystem --
    void bindEngine(const std::shared_ptr<sphb200::Engine>& e) { engine_ = e; }
    const std::shared_ptr<sphb200::Engine>& engine() const { return engine_; }

protected:
    DArray<float3> pos;
    DArray<float3> vel;
    std::shared_ptr<sphb200::Engine> engine_;
    int activeCount_ = -1;
};

// ---- SPHParticles.h:20-60 ---------------------------------------------------------------------
class SPHParticles final : public Particles {
public:
    explicit SPHParticles(const std::vector<float3>& p)
        : Particles(p), pressure(p.size()), density(p.size()), mass(p.size()), particle2Cell(p.size()) {}
    // addition: `capacity` slots with size() == p.size() (a fluid set whose count changes: open boundaries)
    SPHParticles(const std::vector<float3>& p, unsigned int capacity)
        : Particles(p, capacity), pressure(this->capacity()), density(this->capacity()), mass(this->capacity()),
          particle2Cell(this->capacity()) {}
    SPHParticles(const SPHParticles&) = delete;
    SPHParticles& operator=(const SPHParticles&) = delete;
    virtual ~SPHParticles() noexcept {}

    float* getPressurePtr() const { return pressure.addr(); }
    const DArray<float>& getPressure() const { return pressure; }
    float* getDensityPtr() const { return density.addr(); }
    const DArray<float>& getDensity() const { return density; }
    int* getParticle2Cell() const { return particle2Cell.addr(); }
    float* getMassPtr() const { return mass.addr(); }

    // -- addition: this set as the POD the C-ABI takes --
    sphk_particles abi() const {
        sphk_particles p;
        p.pos = reinterpret_cast<float*>(pos.addr()); p.vel = reinterpret_cast<float*>(vel.addr());
        p.mass = mass.addr(); p.density = density.addr(); p.pressure = pressure.addr();
        p.particle2cell = particle2Cell.addr(); p.n = static_cast<int>(size());
        return p;
    }

protected:
    DArray<float> pressure;
    DArray<float> density;
    DArray<float> mass;
    DArray<int> particle2Cell;   // lookup key, left in pre-sort order by the neighbour search (Q2)
};

// ---- BaseSolver.h:20-31 -----------------------------------------------------------------------
class BaseSolver {
public:
    virtual void step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                      const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                      int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float stiff,
                      float visc, float3 G, float surfaceTensionIntensity, float airPressure) = 0;
    virtual ~BaseSolver() {}
protected:
    virtual void advect(std::shared_ptr<SPHParticles>& fluids, float dt, float3 spaceSize) = 0;
    virtual void force(std::shared_ptr<SPHParticles>& fluids, float dt, float3 G) = 0;
};

// ---- BasicSPHSolver.h:20-51 (WCSPH; also the base of DFSPH and PBD) ----------------------------
class BasicSPHSolver : public BaseSolver {
public:
    explicit BasicSPHSolver(int num) : bufferFloat3(num), bufferColorGrad(num), num_(num) {}
    // addition: false = one kernel per reference launch site (the per-op C-ABI path); true (default) = fused sweeps
    void setFusedSweeps(bool on) { if (on != fusedSweeps_) ++configEpoch_; fusedSweeps_ = on; }
    // addition: vorticity confinement (sphk_vorticity_confinement) with strength eps in every step; 0 (default) = off, the
    // reference's step.  Negative or NaN eps is refused (printed, setting kept).  The two buffers it needs are allocated on
    // the first enable.
    void setVorticityConfinement(float eps);
    float vorticityConfinement() const { return vortEps_; }
    // addition: implicit viscosity (sphk_implicit_viscosity; DESIGN.md section 2.5) in every step, on top of the reference's
    // explicit `visc` term: kinematic viscosity nu of the fluid and nuBoundary against walls and bodies (0: free slip), solved
    // to |b - A v|_M <= tol |b|_M or maxIter CG iterations.  nu = 0 (default) = off, the reference's step.  nu or nuBoundary
    // < 0 or NaN, tol <= 0 or NaN, maxIter outside [1, SPHK_IMPLICIT_VISCOSITY_MAX_ITER], and nuBoundary > 0 in a system with
    // dynamic bodies are refused (printed, setting kept).  Every one of the maxIter iterations is enqueued (the ones after
    // convergence return at once), so maxIter should stay near what the scene needs.  The workspace is allocated on the first
    // enable.
    void setImplicitViscosity(float nu, float nuBoundary = 0.0f, float tol = 1e-4f, int maxIter = 20);
    float implicitViscosity() const { return implNu_; }
    // iterations and final relative residual of the last solve (0 before the first); synchronise
    int lastViscosityIterations() const;
    float lastViscosityResidual() const;
    // addition: true when step() enqueues the same kernel sequence every call and never synchronises the host.
    // Only the three shipped solver types can say so: a user-derived solver (the reference API allows subclassing
    // BasicSPHSolver) has per-step host logic of its own, so it is never captured into a step graph.
    virtual bool stepIsGraphSafe() const { return typeid(*this) == typeid(BasicSPHSolver) && !fieldHook_; }
    // addition: bumped whenever a setting that changes the kernel sequence is modified (invalidates a captured graph)
    unsigned int configEpoch() const { return configEpoch_; }
    // additions for the multi-GPU system (SlabSPHSystem): the solver classes stay what they are; after every sweep whose
    // output a later sweep gathers from neighbours the solver tells the system, which refreshes that field on its ghost
    // particles.  what: 1 = velocities, 2 = neighbour scalar (stiffness / lambda), 4 = positions, 0 = any other
    // per-particle array (width 1 or 3 floats).  Unset on one GPU (no calls, no cost).
    using FieldHook = std::function<void(int what, float* array, int width)>;
    using ReduceHook = std::function<double(double)>;
    void setFieldHook(FieldHook h) { fieldHook_ = std::move(h); ++configEpoch_; }
    using RangeHook = std::function<void(int& begin, int& count)>;
    void setReduceHook(ReduceHook h, long long globalCount, RangeHook owned) { reduceHook_ = std::move(h); globalCount_ = globalCount; ownedRange_ = std::move(owned); }
    // the per-particle history array that must travel with a particle when it changes rank (nullptr: none)
    virtual float* historyArray(int& width) { width = 0; return nullptr; }
    // addition: the particle count the solver's buffers hold (its constructor's num)
    int capacity() const { return num_; }
    // addition: the dt an emitted particle's history slot is written with when the coming step runs at dt (PBD: its last predict's)
    virtual float historyTimeStep(float dt) const { return dt; }
    virtual ~BasicSPHSolver() noexcept {}
    virtual void step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                      const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                      int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float stiff,
                      float visc, float3 G, float surfaceTensionIntensity, float airPressure) override;
protected:
    virtual void force(std::shared_ptr<SPHParticles>& fluids, float dt, float3 G) override final;
    virtual void advect(std::shared_ptr<SPHParticles>& fluids, float dt, float3 spaceSize) override final;
    virtual void project(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                         const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float rho0,
                         float stiff, int3 cellSize, float cellLength, float radius, float dt);
    virtual void diffuse(std::shared_ptr<SPHParticles>& fluids, const DArray<int>& cellStartFluid, int3 cellSize,
                         float cellLength, float rho0, float radius, float visc, float dt);
    virtual void handleSurface(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                               const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float rho0,
                               float rhoB, int3 cellSize, float cellLength, float radius, float dt,
                               float surfaceTensionIntensity, float airPressure);
    // the scene of the step in flight (set by step(); the protected hooks above only receive pieces of it)
    struct StepScene {
        sphk_ctx* ctx = nullptr;
        sphk_scene abi{};
    };
    StepScene current_;
    // fused replacements of {computeDensity | computeDensityAlpha} + colour gradient, and viscosity + surface
    void densityAndColorGrad(float* alphaOrNull, float rho0, float rhoB, bool surface);
    void diffuseAndSurface(float rho0, float rhoB, float visc, float dt, float surfaceTensionIntensity, float airPressure,
                           bool surface, bool colorGradReady);
    bool fusedSweeps_ = true;
    unsigned int configEpoch_ = 0;
    FieldHook fieldHook_;
    ReduceHook reduceHook_;
    RangeHook ownedRange_;
    long long globalCount_ = -1;
    void produced(int what, float* array, int width) { if (fieldHook_) fieldHook_(what, array, width); }
    void producedVel(const std::shared_ptr<SPHParticles>& f) { if (fieldHook_) fieldHook_(1, reinterpret_cast<float*>(f->getVelPtr()), 3); }
    float* colorGradBuffer() const { return reinterpret_cast<float*>(bufferColorGrad.addr()); }
    bool beginStep(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                   const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float radius,
                   bool neighborList, int listSkinPermille);
    // vorticity confinement: on when vortEps_ > 0.  vorticity() forms omega (call it before the viscosity / XSPH sweep reads
    // the velocities), confine() applies it (after the surface sweep)
    bool vorticityOn() const { return vortEps_ > 0.0f; }
    float* omegaBuffer() const { return reinterpret_cast<float*>(omega_->addr()); }
    float* omegaNormBuffer() const { return omegaNorm_->addr(); }
    void vorticity(float rho0);
    void confine(const std::shared_ptr<SPHParticles>& fluids, float rho0, float dt);
    // implicit viscosity: on when implNu_ > 0; runs where confine() would run, before it
    bool implicitViscosityOn() const { return implNu_ > 0.0f; }
    void implicitViscosity(const std::shared_ptr<SPHParticles>& fluids, float rho0, float rhoB, float dt);
    // two-way coupled bodies: the reaction of the sweep just run, with its c (sphk_bodies_react); nothing without dynamic bodies
    void react(float c) { if (reacting_) sphb200::check(sphk_bodies_react(current_.ctx, &current_.abi, c), "sphk_bodies_react"); }
    bool reacting_ = false;
private:
    DArray<float3> bufferFloat3;   // viscosity deltaV, then colour gradient (BasicSPHSolver.h:43)
    DArray<float3> bufferColorGrad;   // addition: the fused viscosity+surface sweep needs both at once
    const int num_;
    float vortEps_ = 0.0f;
    std::unique_ptr<DArray<float3>> omega_;      // vorticity omega
    std::unique_ptr<DArray<float>> omegaNorm_;   // |omega|, the neighbour scalar of the confinement sweep
    float implNu_ = 0.0f, implNuB_ = 0.0f, implTol_ = 1e-4f;
    int implMaxIter_ = 20;
    std::unique_ptr<DArray<float>> viscWork_;    // workspace of sphk_implicit_viscosity
    void viscStats(int& iters, float& residual) const;
};

// ---- DFSPHSolver.h:20-64 ----------------------------------------------------------------------
class DFSPHSolver final : public BasicSPHSolver {
public:
    explicit DFSPHSolver(int num, float defaultDensityErrorThreshold = 1e-3f,
                         float defaultDivergenceErrorThreshold = 1e-3f, int defaultMaxIter = 20)
        : BasicSPHSolver(num), alpha(num), bufferFloat(num), bufferInt(num), error(num), denWarmStiff(num),
          densityErrorThreshold(defaultDensityErrorThreshold),
          divergenceErrorThreshold(defaultDivergenceErrorThreshold), maxIter(defaultMaxIter) {}
    virtual ~DFSPHSolver() noexcept {}
    virtual void step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                      const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                      int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float stiff,
                      float visc, float3 G, float surfaceTensionIntensity, float airPressure) override;
    // fixed iteration counts (negative thresholds, Q11), or loop tests evaluated on the device: either way the step is a
    // fixed launch sequence without host synchronisation
    bool stepIsGraphSafe() const override {
        return !fieldHook_ && (deviceLoops_ || (densityErrorThreshold < 0.0f && divergenceErrorThreshold < 0.0f));
    }
    float* historyArray(int& width) override { width = 1; return denWarmStiff.addr(); }
    // addition: false = the reference's host loop (one error sum read back per iteration, DFSPHSolver.cu:206,360)
    void setDeviceLoops(bool on) { if (on != deviceLoops_) ++configEpoch_; deviceLoops_ = on; }
    int lastDivergenceIterations() const { return loopIterations(0, itDiv_); }   // addition: iteration counts of the last step
    int lastDensityIterations() const { return loopIterations(1, itDen_); }
protected:
    // density-error correction with warm start (DFSPHSolver.cu:160-210); hides BasicSPHSolver::project
    virtual int project(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                        const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float rho0,
                        int3 cellSize, float cellLength, float radius, float dt, float errorThreshold, int maxIter);
private:
    int correctDivergenceError(float rho0, float dt, float errorThreshold, int maxIter, int num, bool firstErrorDone);
    float reduceError(int num);
    DArray<float> alpha;
    DArray<float> bufferFloat;     // the stiffness kappa of the paper
    DArray<int> bufferInt;         // kept for layout parity; the re-sort it served is sphk_permute now
    DArray<float> error;
    DArray<float> denWarmStiff;
    const float densityErrorThreshold;
    const float divergenceErrorThreshold;
    const int maxIter;
    int itDiv_ = 0, itDen_ = 0;      // -1: the count lives on the device (read back on demand)
    bool deviceLoops_ = true;
    int loopIterations(int slot, int hostCount) const;
};

// ---- PBDSolver.h:20-85 ------------------------------------------------------------------------
class PBDSolver final : public BasicSPHSolver {
public:
    explicit PBDSolver(int num, int defaultMaxIter = 20, float defaultXSPH_c = 0.05f, float defaultRelaxation = 0.75f)
        : BasicSPHSolver(num), maxIter(defaultMaxIter), xSPH_c(defaultXSPH_c), relaxation(defaultRelaxation),
          bufferInt(num), fluidPosLast(num), bufferFloat3(num), bufferFloat(num) {}
    explicit PBDSolver(const std::shared_ptr<SPHParticles>& particles, int defaultMaxIter = 20,
                       float defaultXSPH_c = 0.1f, float defaultRelaxation = 1.0f)
        : BasicSPHSolver(particles->size()), maxIter(defaultMaxIter), xSPH_c(defaultXSPH_c),
          relaxation(defaultRelaxation), bufferInt(particles->size()), fluidPosLast(particles->size()),
          bufferFloat3(particles->size()), bufferFloat(particles->size()) {
        initializePosLast(particles->getPos());
    }
    virtual ~PBDSolver() noexcept {}
    virtual void step(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                      const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float3 spaceSize,
                      int3 cellSize, float cellLength, float radius, float dt, float rho0, float rhoB, float stiff,
                      float visc, float3 G, float surfaceTensionIntensity, float airPressure) override;
    bool stepIsGraphSafe() const override { return posLastInitialized && !fieldHook_; }
    float* historyArray(int& width) override { width = 3; return reinterpret_cast<float*>(fluidPosLast.addr()); }
    float historyTimeStep(float dt) const override { return lastPredictDt_ > 0.0f ? lastPredictDt_ : dt; }
    void initializePosLast(const DArray<float3>& posFluid) {
        CUDA_CALL(cudaMemcpy(fluidPosLast.addr(), posFluid.addr(), sizeof(float3) * std::min(fluidPosLast.length(), posFluid.length()),
                             cudaMemcpyDeviceToDevice));
        posLastInitialized = true;
    }
protected:
    void predict(std::shared_ptr<SPHParticles>& fluids, float dt, float3 spaceSize);
    virtual int project(std::shared_ptr<SPHParticles>& fluids, const std::shared_ptr<SPHParticles>& boundaries,
                        const DArray<int>& cellStartFluid, const DArray<int>& cellStartBoundary, float rho0,
                        int3 cellSize, float3 spaceSize, float cellLength, float radius, int maxIter);
    virtual void diffuse(std::shared_ptr<SPHParticles>& fluids, const DArray<int>& cellStartFluid, int3 cellSize,
                         float cellLength, float rho0, float radius, float visc);
private:
    void updateNeighborhood(const std::shared_ptr<SPHParticles>& particles);
    float reactCoef_ = 0.0f;       // 1 / (rho0 dt) of the step in flight: c of the position-correction reaction
    // the dt of the last predict: the projection and the velocity derivation of the next step act on the interval it advanced
    // (0: none yet, the step's own dt is used)
    float lastPredictDt_ = 0.0f;
    bool posLastInitialized = false;
    const int maxIter;
    const float xSPH_c;
    const float relaxation;
    DArray<int> bufferInt;
    DArray<float3> fluidPosLast;
    DArray<float3> bufferFloat3;   // delta-pos buffer; shadows the base-class buffer like the reference (Q13)
    DArray<float> bufferFloat;     // lambda
};

// ---- SPHSystem.h:20-83 ------------------------------------------------------------------------
class SPHSystem {
public:
    SPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
              std::shared_ptr<BaseSolver>& solver, float3 spaceSize, float sphCellLength, float sphSmoothingRadius,
              float dt, float sphM0, float sphRho0, float sphRhoBoundary, float sphStiff, float sphVisc,
              float sphSurfaceTensionIntensity, float sphAirPressure, float3 sphG, int3 cellSize);
    // addition: the same system with kinematic rigid bodies.  The boundary set becomes the caller's (static) boundary
    // particles followed by the bodies' particles, in the order given: getBoundaries() and boundarySize() include the body
    // particles.  Every step() moves the bodies (pose update, placement, boundary search) before the fluid search.  An empty
    // vector is the constructor above.
    SPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
              std::shared_ptr<BaseSolver>& solver, float3 spaceSize, float sphCellLength, float sphSmoothingRadius,
              float dt, float sphM0, float sphRho0, float sphRhoBoundary, float sphStiff, float sphVisc,
              float sphSurfaceTensionIntensity, float sphAirPressure, float3 sphG, int3 cellSize,
              const std::vector<sphb200::KinematicBody>& bodies);
    // addition: the same system with open boundaries (DESIGN.md section 2.6): every step() removes the fluid particles inside a
    // sink, emits the layers the emitters' schedules ask for into the free slots of the fluid set (fluidParticles' capacity),
    // and runs the solver on the live particles.  Such a system never captures a step graph.  Refused with a printed message,
    // building the closed system (openBoundariesActive() false): a solver that is not a BasicSPHSolver or whose buffers hold
    // fewer particles than the fluid's capacity, an invalid emitter or sink, more than 16 of either, and an emitter whose layer
    // (or the layer advanced by speed * dt) reaches outside the clamp box [0, 0.99 spaceSize].  Empty vectors are the
    // constructors above.
    SPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
              std::shared_ptr<BaseSolver>& solver, float3 spaceSize, float sphCellLength, float sphSmoothingRadius,
              float dt, float sphM0, float sphRho0, float sphRhoBoundary, float sphStiff, float sphVisc,
              float sphSurfaceTensionIntensity, float sphAirPressure, float3 sphG, int3 cellSize,
              const std::vector<sphb200::KinematicBody>& bodies, const sphb200::OpenBoundaries& open);
    SPHSystem(const SPHSystem&) = delete;
    SPHSystem& operator=(const SPHSystem&) = delete;
    ~SPHSystem() noexcept;

    float step();   // neighbour search + solver step; returns the step's milliseconds (SPHSystem.cu:129-158)

    int size() const { return fluidSize(); }
    int fluidSize() const { return static_cast<int>(_fluids->size()); }
    int boundarySize() const { return static_cast<int>(_boundaries->size()); }
    int totalSize() const { return fluidSize() + boundarySize(); }
    auto getFluids() const { return static_cast<const std::shared_ptr<SPHParticles>>(_fluids); }
    auto getBoundaries() const { return static_cast<const std::shared_ptr<SPHParticles>>(_boundaries); }

    // -- additions --
    const DArray<int>& getCellStartFluid() const { return cellStartFluid; }
    const DArray<int>& getCellStartBoundary() const { return cellStartBoundary; }
    const std::shared_ptr<sphb200::Engine>& engine() const { return _engine; }
    void setStepGraph(bool on);   // replay each step as one CUDA graph when the solver allows it (default on)
    bool stepGraphActive() const { return _graphExec != nullptr; }   // the next step replays a captured graph
    // kinematic bodies: a new motion takes effect at the next step() (an asynchronous copy; a captured step graph stays
    // valid).  getBodyPose synchronises.  Both print and ignore an out-of-range body index.
    int bodyCount() const { return static_cast<int>(_bodyMotion.size() / 6); }
    void setBodyMotion(int body, float3 linearVelocity, float3 angularVelocity);
    void getBodyPose(int body, float3& position, float4& orientation) const;
    // two-way coupled bodies (any body with mass > 0): the current motion (the integrated one for a dynamic body), and the
    // {J, H} the fluid gave a body over the last step (held bodies included; zero without dynamic bodies).  Both synchronise
    // and print and ignore an out-of-range body index.
    void getBodyMotion(int body, float3& linearVelocity, float3& angularVelocity) const;
    void getBodyImpulse(int body, float3& linearImpulse, float3& angularImpulse) const;
    bool bodiesDynamic() const { return _bodiesDynamic; }   // the dynamics were declared (false if the engine refused them)
    // open boundaries: cumulative {emitted, removed, refused} particle counts, and whether the system has emitters or sinks
    sphb200::OpenBoundaryStats openBoundaryStats() const { return _openStats; }
    bool openBoundariesActive() const { return _open; }
    // the sticky bits of the per-step count check (sphk_open_check; 0 = every step's in-grid count matched; synchronises)
    int openBoundaryCheck() const;
    // CFL-adaptive time stepping (DESIGN.md section 2.8): from the next step on, every step() runs at the dt of the rule
    // sphk_time_step {C, dtMin, dtMax, R = sphSmoothingRadius, |G|} applied to the speed bound the previous step left on the
    // device (fluid, bodies and the emitters' speeds).  0 = the default: dtMax = the constructor's dt, dtMin = dtMax / 64.
    // C <= 0, a non-finite value, a negative one, dtMin > dtMax, and for a system with emitters a dtMax above the constructor's dt
    // (the emitters were checked against the clamp box for that dt) are refused (printed, setting kept, false returned).  An adaptive
    // system runs plain launches and never captures a step graph; disableAdaptiveTimeStep() returns to the constructor's dt and
    // allows it again.
    bool setAdaptiveTimeStep(float C, float dtMin = 0.0f, float dtMax = 0.0f);
    void disableAdaptiveTimeStep();
    bool adaptiveTimeStep() const { return _adaptive; }
    // the next step's dt is chosen from the speed bound measured at the end of the previous step (or by setAdaptiveTimeStep).
    // setBodyMotion measures it again; a caller that writes velocities or positions through the raw accessors between steps
    // calls refreshSpeedBound() so that the next dt sees them (no effect on a system that is not adaptive)
    void refreshSpeedBound();
    // CFL substeps until frameSeconds (> 0) of simulated time have passed (the last one is shortened to end the frame exactly, the
    // one before it halved when the frame would otherwise end with a sliver); returns their count (0 and a printed message for a
    // system that is not adaptive or a frame that is not finite and > 0)
    int advance(double frameSeconds);
    float lastTimeStep() const { return _lastDt; }            // the dt of the last step
    double simulatedTime() const { return _simTime; }         // the double sum of the float dt of every step
    sphb200::AdaptiveStats adaptiveStats() const { return _adaptiveStats; }

private:
    std::shared_ptr<SPHParticles> _fluids;
    const std::shared_ptr<SPHParticles> _boundaries;
    std::shared_ptr<BaseSolver> _solver;
    DArray<int> cellStartFluid;
    DArray<int> cellStartBoundary;
    const float3 _spaceSize;
    const float _sphSmoothingRadius;
    const float _sphCellLength;
    const float _dt;
    const float _sphRho0;
    const float _sphRhoBoundary;
    const float _sphStiff;
    const float3 _sphG;
    const float _sphVisc;
    const float _sphSurfaceTensionIntensity;
    const float _sphAirPressure;
    const int3 _cellSize;
    std::shared_ptr<sphb200::Engine> _engine;
    cudaEvent_t _evStart = nullptr, _evStop = nullptr;
    // CUDA graph of one whole step (fixed-iteration solvers only: the kernel sequence is then the same every step)
    cudaGraphExec_t _graphExec = nullptr;
    long long _graphLaunches = 0;
    unsigned int _graphConfigEpoch = 0;   // solver configEpoch() the graph was captured with
    int _plainSteps = 0;
    bool _graphEnabled = true;
    bool solverIsGraphSafe() const;
    unsigned int solverConfigEpoch() const;
    void dropStepGraph();
    std::vector<float> _bodyMotion;       // host copy of all bodies' motions (6 floats each); empty: no bodies
    bool _bodiesDynamic = false;          // some body has mass > 0: sphk_bodies_integrate ends every step
    void computeBoundaryMass();
    void searchForStep();                 // bodies (if any), then the fluid search
    void integrateBodies();               // sphk_bodies_integrate at the end of a step with dynamic bodies
    void neighborSearch(const std::shared_ptr<SPHParticles>& particles, DArray<int>& cellStart);
    // open boundaries
    bool _open = false;
    float _sphM0 = 0.0f;
    std::vector<sphk_emitter> _emitters;
    std::vector<double> _emitterCarry;    // the schedule's carry of each emitter (sphk_emitter_advance)
    std::vector<float> _sinkBoxes;        // {lo.xyz, hi.xyz} per sink
    std::vector<float> _layerOffsets;     // scratch of sphk_emitter_advance
    sphb200::OpenBoundaryStats _openStats;
    const char* openRefusal(const sphb200::OpenBoundaries& open) const;
    int openEmit(int n);                  // sinks and emitters before the search; returns the emitted count
    // time steps: every kernel of a step receives _stepDt (the constructor's dt unless adaptive)
    float _stepDt = 0.0f, _lastDt = 0.0f;
    double _simTime = 0.0;
    bool _adaptive = false;
    sphk_time_step_rule _rule{};
    sphb200::AdaptiveStats _adaptiveStats;
    float runStep();                      // one step at _stepDt
    float chooseTimeStep(double remaining, bool& frameEnd);   // waits for the last speed bound, applies the rule
    void measureSpeed();                  // enqueues the speed bound of the current state (sphk_step_speed)
};

// ---- vbo.cu:46-51 --------------------------------------------------------------------------------
// Same signature and linkage as the reference's render hook; writes plain device buffers (the reference maps a GL
// vertex buffer and passes its device pointers: the call site main.cpp:268-281 is unchanged).
extern "C" void generate_dots(float3* dot, float3* color, const std::shared_ptr<SPHParticles> particles);
