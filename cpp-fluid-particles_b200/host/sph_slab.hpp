// sph_slab.hpp -- SlabSPHSystem: SPHSystem sharded over the GPUs of one box, behind the same class API.
//
// The reference (SPHSystem.h:20-83) is single-GPU.  SlabSPHSystem takes the SAME constructor arguments as SPHSystem -- the
// global particle sets, a solver object constructed exactly as at the reference call site (main.cpp:119-130), the 13 scene
// parameters -- plus the rank's place among the processes of the job (one process per GPU).  The three solver classes are used
// unchanged: the system owns the decomposition (x-slabs of cell planes: contiguous key ranges, CUDAFunctions.cuh:68; halo = one
// plane), the once-per-step candidate exchange + search of [ghost-left | owned | ghost-right], and -- through the solvers'
// field hook -- the refresh of every field a sweep produced on the ghost particles (peer-memory mailbox halos / NCCL,
// csrc/sphk_mg.cu).  Host side only (g++); everything on the device goes through the C-ABI.  python's slabs.SlabSystem is the
// same algorithm over torch tensors (it drives bench.py --gpus N and carries the host-free step assembly); this class is the
// drop-in for C++ callers.
#pragma once

#include <string>

#include "sph_api.hpp"

namespace sphb200 {
// Where this process sits in the job.  The ranks of one node find each other through files in `rendezvousDir` (a directory
// that is fresh for every run): the NCCL id of rank 0 and the CUDA IPC handles of the halo mailboxes are exchanged there.
struct SlabBootstrap {
    int rank = 0;
    int world = 1;
    std::string rendezvousDir;
    double timeoutSeconds = 120.0;
};
}  // namespace sphb200

class SlabSPHSystem {
public:
    SlabSPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
                  std::shared_ptr<BaseSolver>& solver, float3 spaceSize, float sphCellLength, float sphSmoothingRadius, float dt,
                  float sphM0, float sphRho0, float sphRhoBoundary, float sphStiff, float sphVisc, float sphSurfaceTensionIntensity,
                  float sphAirPressure, float3 sphG, int3 cellSize, const sphb200::SlabBootstrap& boot);
    SlabSPHSystem(const SlabSPHSystem&) = delete;
    SlabSPHSystem& operator=(const SlabSPHSystem&) = delete;
    ~SlabSPHSystem() noexcept;

    // candidate exchange + neighbour search + solver step of this rank; milliseconds like SPHSystem::step.  Collective: every rank
    // calls it.  Throws std::runtime_error when this rank cannot keep the decomposition's contracts (capacity exceeded, ghost planes
    // that do not match the neighbours', a halo that did not arrive): end the process then -- the other ranks wait for this one.
    float step();

    bool ok() const { return ok_; }
    // probes and gauges are single-context only (a probe near a cut would miss the other rank's fluid): refused, printed
    bool setProbes(const sphb200::Probes&) {
        printf("SlabSPHSystem: probes and gauges are not supported on slab ranks (single-GPU SPHSystem only)\n");
        return false;
    }
    // checkpoints are single-context only (DESIGN.md section 2.14): refused, printed
    bool checkpoint(const std::string&, const std::vector<unsigned char>& = {}) {
        printf("SlabSPHSystem: checkpoints are not supported on slab ranks (single-GPU SPHSystem only)\n");
        return false;
    }
    bool restore(const std::string&, std::vector<unsigned char>* = nullptr) {
        printf("SlabSPHSystem: checkpoints are not supported on slab ranks (single-GPU SPHSystem only)\n");
        return false;
    }
    int size() const { return nOwn_; }                  // particles this rank owns
    int ownedBegin() const { return ownBegin_; }        // ... stored at [ownedBegin, ownedBegin + size) of the local set
    int globalSize() const { return nGlobal_; }
    int rank() const { return boot_.rank; }
    int world() const { return boot_.world; }
    // the LOCAL set [ghost-left | owned | ghost-right] (sorted by local cell index) and the local boundary set
    auto getFluids() const { return static_cast<const std::shared_ptr<SPHParticles>>(fluids_); }
    auto getBoundaries() const { return static_cast<const std::shared_ptr<SPHParticles>>(boundaries_); }
    int straysRouted();                                 // strays all ranks collected for the last step (synchronises; introspection)
    const char* haloTransport() const { return transport_ == 1 ? "peer-memory mailboxes" : "NCCL send/recv"; }
    // the same setter as SPHSystem's; not supported on slab ranks (the speed bound would need a global maximum): step() throws
    void setAdaptiveTimeStep(float, float = 0.0f, float = 0.0f) { adaptive_ = true; }
    void disableAdaptiveTimeStep() { adaptive_ = false; }

private:
    bool adaptive_ = false;
    struct Ranges { int own[2], toLeft[2], toRight[2], first[2], last[2], ghostL[2], ghostR[2]; };
    void beginStep();
    void searchAll(int n);
    void readBounds(int b[8]);
    static Ranges planeRanges(const int b[8], int w);
    void halo(int what, float* array, int width);
    bool rendezvous();
    sphk_scene scene() const;

    sphb200::SlabBootstrap boot_;
    bool ok_ = false;
    std::shared_ptr<SPHParticles> fluids_, boundaries_;
    std::shared_ptr<BaseSolver> solver_;
    std::shared_ptr<sphb200::Engine> engine_;
    sphk_mg_comm* comm_ = nullptr;
    int transport_ = 0;
    std::unique_ptr<DArray<int>> csF_, csB_;
    std::unique_ptr<DArray<float3>> altPos_, altVel_;
    std::unique_ptr<DArray<float>> altHist_;
    int* dBounds_ = nullptr;          // device: the 8 plane offsets gathered from csF_
    // strays (include/sphk.h): particles that crossed two or more planes in a step are routed to every rank
    int strayCap_ = 0;                // per rank and step; SPHK_SLAB_STRAYS (default 2048, 0 = off)
    float *strayBlock_ = nullptr, *strayGathered_ = nullptr;
    bool strayPending_ = false;
    void collectStrays();
    int x0_ = 0, x1_ = 0, w_ = 0, planeCells_ = 0, cap_ = 0, nGlobal_ = 0;
    int nOwn_ = 0, ownBegin_ = 0, nGhostL_ = 0, nGhostR_ = 0;
    bool haveRanges_ = false;
    Ranges r_{};
    int candFrom_[2] = {0, 0};
    int haloRanges_[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const float3 spaceSize_;
    const float radius_, cellLength_, dt_, rho0_, rhoB_, stiff_, visc_, surfaceTension_, airPressure_;
    const float3 G_;
    int3 localCellSize_;
    cudaEvent_t evStart_ = nullptr, evStop_ = nullptr;
};
