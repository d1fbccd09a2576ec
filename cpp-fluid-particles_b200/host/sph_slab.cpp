// sph_slab.cpp -- SlabSPHSystem: the class-API system sharded by x-slabs over the GPUs of one box (see sph_slab.hpp).
// Host orchestration only (g++); the algorithm is the one of cpp-fluid-particles_b200/slabs.py (module docstring there):
// one candidate exchange + one search per step, ownership decided by the sort, a halo after every sweep whose output the
// next sweep gathers from neighbours.  No reference counterpart (the reference is single-GPU, SURVEY 8e).
#include "sph_slab.hpp"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

using sphb200::check;

namespace {

// ---- tiny file rendezvous (ranks of one node, fresh directory per run) -------------------------------------------------
bool write_file_atomic(const std::string& path, const void* data, size_t bytes) {
    const std::string tmp = path + ".tmp";
    {
        std::ofstream f(tmp, std::ios::binary | std::ios::trunc);
        if (!f) return false;
        f.write(static_cast<const char*>(data), static_cast<std::streamsize>(bytes));
        if (!f) return false;
    }
    return std::rename(tmp.c_str(), path.c_str()) == 0;
}

bool read_file_wait(const std::string& path, void* data, size_t bytes, double timeoutSeconds) {
    const auto t0 = std::chrono::steady_clock::now();
    for (;;) {
        std::ifstream f(path, std::ios::binary);
        if (f) {
            f.read(static_cast<char*>(data), static_cast<std::streamsize>(bytes));
            if (f.gcount() == static_cast<std::streamsize>(bytes)) return true;
        }
        if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > timeoutSeconds) return false;
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
    }
}

// slabs.choose_cuts: plane indices X_0 = 0 < X_1 < ... < X_world = n_planes balancing the particle counts
std::vector<int> choose_cuts(const std::vector<long long>& countPerPlane, int world) {
    const int nPlanes = static_cast<int>(countPerPlane.size());
    std::vector<long long> cdf(nPlanes);
    long long acc = 0;
    for (int p = 0; p < nPlanes; ++p) { acc += countPerPlane[p]; cdf[p] = acc; }
    const long long total = acc;
    std::vector<int> cuts{0};
    for (int g = 1; g < world; ++g) {
        const double target = static_cast<double>(total) * g / world;
        int x = static_cast<int>(std::lower_bound(cdf.begin(), cdf.end(), target,
                                                  [](long long a, double t) { return static_cast<double>(a) < t; }) - cdf.begin()) + 1;
        x = std::max(x, cuts.back() + 1);
        x = std::min(x, nPlanes - (world - g));
        cuts.push_back(x);
    }
    cuts.push_back(nPlanes);
    return cuts;
}

// a rank that cannot keep the decomposition's contracts must not go on (its neighbours would compute with stale ghosts or wait for
// it): the step throws, the caller ends the process, the launcher ends the job
[[noreturn]] void fail(int rank, const std::string& what) {
    throw std::runtime_error("SlabSPHSystem: rank " + std::to_string(rank) + ": " + what);
}

}  // namespace

// slabs.plane_ranges: from the plane offsets (s0, s1, s2, s3, s_{w-1}, s_w, s_{w+1}, s_end) of a sorted local set
SlabSPHSystem::Ranges SlabSPHSystem::planeRanges(const int b[8], int w) {
    const int s0 = b[0], s1 = b[1], s2 = b[2], s3 = b[3], swm1 = b[4], sw = b[5], sw1 = b[6], send = b[7];
    Ranges r;
    r.own[0] = s1; r.own[1] = sw1;
    r.toLeft[0] = s1; r.toLeft[1] = w >= 2 ? std::min(s3, sw1) : sw1;
    r.toRight[0] = w >= 2 ? std::max(swm1, s1) : s1; r.toRight[1] = sw1;
    r.first[0] = s1; r.first[1] = w >= 2 ? s2 : sw1;
    r.last[0] = w >= 2 ? sw : s1; r.last[1] = sw1;
    r.ghostL[0] = s0; r.ghostL[1] = s1;
    r.ghostR[0] = sw1; r.ghostR[1] = send;
    return r;
}

SlabSPHSystem::SlabSPHSystem(std::shared_ptr<SPHParticles>& fluidParticles, std::shared_ptr<SPHParticles>& boundaryParticles,
                             std::shared_ptr<BaseSolver>& solver, const float3 spaceSize, const float sphCellLength,
                             const float sphSmoothingRadius, const float dt, const float sphM0, const float sphRho0,
                             const float sphRhoBoundary, const float sphStiff, const float sphVisc,
                             const float sphSurfaceTensionIntensity, const float sphAirPressure, const float3 sphG,
                             const int3 cellSize, const sphb200::SlabBootstrap& boot)
    : boot_(boot), solver_(std::move(solver)), spaceSize_(spaceSize), radius_(sphSmoothingRadius), cellLength_(sphCellLength), dt_(dt),
      rho0_(sphRho0), rhoB_(sphRhoBoundary), stiff_(sphStiff), visc_(sphVisc), surfaceTension_(sphSurfaceTensionIntensity),
      airPressure_(sphAirPressure), G_(sphG), localCellSize_{0, cellSize.y, cellSize.z} {
    // the caller's shared_ptrs are moved from, as SPHSystem does (SPHSystem.cu:50-51)
    std::shared_ptr<SPHParticles> globalFluids = std::move(fluidParticles);
    std::shared_ptr<SPHParticles> globalBoundaries = std::move(boundaryParticles);
    auto* known = dynamic_cast<BasicSPHSolver*>(solver_.get());
    if (!known) { printf("SlabSPHSystem: the solver must derive from BasicSPHSolver (field hooks)\n"); return; }
    if (boot_.world < 1 || boot_.rank < 0 || boot_.rank >= boot_.world) { printf("SlabSPHSystem: bad rank / world\n"); return; }
    CUDA_CALL(cudaEventCreate(&evStart_));
    CUDA_CALL(cudaEventCreate(&evStop_));
    nGlobal_ = static_cast<int>(globalFluids->size());
    const int cx = cellSize.x, cy = cellSize.y, cz = cellSize.z;
    planeCells_ = cy * cz;

    // ---- static partition from the particle CDF along x (host approximation of the hash; a particle one plane off is simply
    // migrated by the first step) -----------------------------------------------------------------------------------------------
    std::vector<float3> hpos(static_cast<size_t>(nGlobal_));
    CUDA_CALL(cudaMemcpy(hpos.data(), globalFluids->getPosPtr(), sizeof(float3) * hpos.size(), cudaMemcpyDeviceToHost));
    std::vector<int> plane(hpos.size());
    std::vector<long long> perPlane(static_cast<size_t>(cx), 0);
    for (size_t i = 0; i < hpos.size(); ++i) {
        int p = static_cast<int>(hpos[i].x / sphCellLength);
        p = std::min(std::max(p, 0), cx - 1);
        plane[i] = p;
        perPlane[static_cast<size_t>(p)]++;
    }
    const std::vector<int> cuts = choose_cuts(perPlane, boot_.world);
    x0_ = cuts[static_cast<size_t>(boot_.rank)]; x1_ = cuts[static_cast<size_t>(boot_.rank) + 1]; w_ = x1_ - x0_;
    std::vector<float3> mine;
    for (size_t i = 0; i < hpos.size(); ++i)
        if (plane[i] >= x0_ && plane[i] < x1_) mine.push_back(hpos[i]);
    const int nMine = static_cast<int>(mine.size());
    if (boot_.world > 1) {
        const char* e = std::getenv("SPHK_SLAB_STRAYS");
        strayCap_ = e ? std::max(std::atoi(e), 0) : 2048;
    }
    // (never above the global count: the solver's own buffers were sized with it at the reference call site, main.cpp:119-130)
    cap_ = std::min(static_cast<int>(std::max<double>(nMine, static_cast<double>(nGlobal_) / boot_.world) * 1.6) + 4096 + boot_.world * strayCap_, nGlobal_);
    mine.resize(static_cast<size_t>(cap_), make_float3(0.f, 0.f, 0.f));
    fluids_ = std::make_shared<SPHParticles>(mine);
    hpos.clear(); hpos.shrink_to_fit(); plane.clear(); plane.shrink_to_fit();

    // ---- boundary: masses from the GLOBAL boundary set (SPHSystem.cu:69-71), then the slice of this rank's planes [x0-1, x1+1)
    std::vector<float3> bpos;
    std::vector<float> bmass;
    {
        const int nb = static_cast<int>(globalBoundaries->size());
        auto tmp = std::make_shared<sphb200::Engine>(1, nb, cellSize, sphCellLength);
        if (!tmp->ok()) return;
        DArray<int> csG(static_cast<unsigned int>(cx * cy * cz + 1));
        const sphk_particles b = globalBoundaries->abi();
        check(sphk_neighbor_search(tmp->ctx(), 1, &b, csG.addr()), "sphk_neighbor_search(global boundary)");
        check(sphk_boundary_mass(tmp->ctx(), &b, csG.addr(), sphRhoBoundary, sphSmoothingRadius), "sphk_boundary_mass");
        check(sphk_synchronize(tmp->ctx()), "sphk_synchronize");
        std::vector<int> planeStart(static_cast<size_t>(cx) + 1);
        CUDA_CALL(cudaMemcpy2D(planeStart.data(), sizeof(int), csG.addr(), sizeof(int) * static_cast<size_t>(planeCells_), sizeof(int),
                               static_cast<size_t>(cx) + 1, cudaMemcpyDeviceToHost));
        const int a = planeStart[static_cast<size_t>(std::max(x0_ - 1, 0))], e = planeStart[static_cast<size_t>(std::min(x1_ + 1, cx))];
        if (e > a) {
            bpos.resize(static_cast<size_t>(e - a)); bmass.resize(static_cast<size_t>(e - a));
            CUDA_CALL(cudaMemcpy(bpos.data(), globalBoundaries->getPosPtr() + a, sizeof(float3) * bpos.size(), cudaMemcpyDeviceToHost));
            CUDA_CALL(cudaMemcpy(bmass.data(), globalBoundaries->getMassPtr() + a, sizeof(float) * bmass.size(), cudaMemcpyDeviceToHost));
        } else {                                    // keep the C-ABI happy: one far-away massless dummy
            bpos.assign(1, make_float3(-1.0e3f, -1.0e3f, -1.0e3f)); bmass.assign(1, 0.0f);
        }
    }
    boundaries_ = std::make_shared<SPHParticles>(bpos);
    CUDA_CALL(cudaMemcpy(boundaries_->getMassPtr(), bmass.data(), sizeof(float) * bmass.size(), cudaMemcpyHostToDevice));
    globalFluids.reset(); globalBoundaries.reset();

    // ---- local context: planes [x0 - 1, x1 + 1) ----------------------------------------------------------------------------------
    localCellSize_ = make_int3(w_ + 2, cy, cz);
    engine_ = std::make_shared<sphb200::Engine>(cap_, static_cast<int>(bpos.size()), localCellSize_, sphCellLength, make_int3(x0_ - 1, 0, 0));
    if (!engine_->ok()) return;
    fluids_->bindEngine(engine_);
    boundaries_->bindEngine(engine_);
    const unsigned int ncellsLocal = static_cast<unsigned int>((w_ + 2) * cy * cz);
    csF_ = std::make_unique<DArray<int>>(ncellsLocal + 1);
    csB_ = std::make_unique<DArray<int>>(ncellsLocal + 1);
    altPos_ = std::make_unique<DArray<float3>>(static_cast<unsigned int>(cap_));
    altVel_ = std::make_unique<DArray<float3>>(static_cast<unsigned int>(cap_));
    altHist_ = std::make_unique<DArray<float>>(static_cast<unsigned int>(3 * cap_));
    CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&dBounds_), 8 * sizeof(int)));
    if (boot_.world > 1 && !rendezvous()) return;

    // ---- SPHSystem.cu:68-76 on the local sets (boundary masses are given: the search only sorts and packs them) -------------------
    check(sphk_fill(engine_->ctx(), fluids_->getMassPtr(), cap_, sphM0), "sphk_fill");
    {
        const sphk_particles b = boundaries_->abi();
        check(sphk_neighbor_search(engine_->ctx(), 1, &b, csB_->addr()), "sphk_neighbor_search(boundary)");
    }
    known->setFieldHook([this](int what, float* array, int width) { halo(what, array, width); });
    known->setReduceHook(
        [this](double x) {
            if (comm_) check(sphk_mg_allreduce_sum(comm_, &x), "sphk_mg_allreduce_sum");
            return x;
        },
        nGlobal_, [this](int& begin, int& count) { begin = ownBegin_; count = nOwn_; });
    nOwn_ = nMine; ownBegin_ = 0;
    fluids_->setActiveCount(nMine);
    ok_ = true;
    step();                                         // the constructor's implicit step 0 (Q3)
}

SlabSPHSystem::~SlabSPHSystem() noexcept {
    if (engine_ && engine_->ok()) sphk_synchronize(engine_->ctx());
    if (comm_) sphk_mg_destroy(comm_);
    if (dBounds_) cudaFree(dBounds_);
    if (strayBlock_) cudaFree(strayBlock_);
    if (strayGathered_) cudaFree(strayGathered_);
    if (evStart_) cudaEventDestroy(evStart_);
    if (evStop_) cudaEventDestroy(evStop_);
}

// NCCL id from rank 0 and the mailbox IPC handles through files in boot_.rendezvousDir; every rank ends up on the same transport
bool SlabSPHSystem::rendezvous() {
    const std::string dir = boot_.rendezvousDir;
    if (dir.empty()) { printf("SlabSPHSystem: rendezvousDir is empty\n"); return false; }
    unsigned char id[128];
    if (boot_.rank == 0) {
        if (sphk_mg_unique_id(id) != 0 || !write_file_atomic(dir + "/nccl_id", id, sizeof(id))) {
            printf("SlabSPHSystem: cannot publish the NCCL id in %s\n", dir.c_str());
            return false;
        }
    } else if (!read_file_wait(dir + "/nccl_id", id, sizeof(id), boot_.timeoutSeconds)) {
        printf("SlabSPHSystem: rank %d: no NCCL id in %s\n", boot_.rank, dir.c_str());
        return false;
    }
    // payload capacity of a mailbox: a function of GLOBAL quantities only (every rank must use the same layout)
    const long long mailbox = 3LL * std::max(262144LL, static_cast<long long>(static_cast<double>(nGlobal_) / boot_.world * 1.6) / 4);
    const int rc = sphk_mg_init(&comm_, boot_.rank, boot_.world, id, engine_->stream(), mailbox);
    if (rc != 0) { printf("SlabSPHSystem: sphk_mg_init failed: %s (%d)\n", sphk_error_string(rc), rc); comm_ = nullptr; return false; }
    // mailbox wiring; the ranks agree on the outcome (mixed transports would wait for each other forever)
    unsigned char mine[64], left[64], right[64];
    unsigned char okMine = sphk_mg_ipc_handle(comm_, mine) == 0 ? 1 : 0;
    write_file_atomic(dir + "/ipc_" + std::to_string(boot_.rank), mine, sizeof(mine));
    const bool hasL = boot_.rank > 0, hasR = boot_.rank < boot_.world - 1;
    if (hasL && !read_file_wait(dir + "/ipc_" + std::to_string(boot_.rank - 1), left, sizeof(left), boot_.timeoutSeconds)) okMine = 0;
    if (hasR && !read_file_wait(dir + "/ipc_" + std::to_string(boot_.rank + 1), right, sizeof(right), boot_.timeoutSeconds)) okMine = 0;
    if (okMine && sphk_mg_ipc_connect(comm_, hasL ? left : nullptr, hasR ? right : nullptr) != 0) okMine = 0;
    write_file_atomic(dir + "/connected_" + std::to_string(boot_.rank), &okMine, 1);
    bool all = true;
    for (int r = 0; r < boot_.world; ++r) {
        unsigned char o = 0;
        if (!read_file_wait(dir + "/connected_" + std::to_string(r), &o, 1, boot_.timeoutSeconds)) o = 0;
        all = all && o == 1;
    }
    transport_ = all ? 1 : 0;
    if (!all && boot_.rank == 0) printf("SlabSPHSystem: peer-memory mailboxes unavailable: NCCL halos instead\n");
    check(sphk_mg_set_transport(comm_, transport_), "sphk_mg_set_transport");
    return true;
}

sphk_scene SlabSPHSystem::scene() const {
    sphk_scene s;
    s.fluid = fluids_->abi();
    s.boundary = boundaries_->abi();
    s.cell_start_fluid = csF_->addr();
    s.cell_start_boundary = csB_->addr();
    s.radius = radius_;
    return s;
}

void SlabSPHSystem::searchAll(int n) {
    fluids_->setActiveCount(n);
    const sphk_particles p = fluids_->abi();
    check(sphk_neighbor_search(engine_->ctx(), 0, &p, csF_->addr()), "sphk_neighbor_search");
}

void SlabSPHSystem::readBounds(int b[8]) {
    const int pc = planeCells_, w = w_;
    const int idx[8] = {0, pc, 2 * pc, 3 * pc, std::max(w - 1, 0) * pc, w * pc, (w + 1) * pc, (w + 2) * pc};
    cudaStream_t st = engine_->stream();
    for (int k = 0; k < 8; ++k)
        CUDA_CALL(cudaMemcpyAsync(dBounds_ + k, csF_->addr(idx[k]), sizeof(int), cudaMemcpyDeviceToDevice, st));
    CUDA_CALL(cudaMemcpyAsync(b, dBounds_, 8 * sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_CALL(cudaStreamSynchronize(st));
}

// one halo of a field the solver has just produced (BasicSPHSolver::FieldHook)
void SlabSPHSystem::halo(int what, float* array, int width) {
    if (!comm_ || boot_.world == 1) return;
    const sphk_scene s = scene();
    check(sphk_mg_halo(comm_, engine_->ctx(), &s, what, array, width, haloRanges_), "sphk_mg_halo");
}

// slabs.SlabSystem._collect_strays: owned particles that crossed two or more planes since the last search leave the regular flow
void SlabSPHSystem::collectStrays() {
    auto* known = dynamic_cast<BasicSPHSolver*>(solver_.get());
    int histWidth = 0;
    float* hist = known->historyArray(histWidth);
    float* live[3] = {reinterpret_cast<float*>(fluids_->getPosPtr()), reinterpret_cast<float*>(fluids_->getVelPtr()), hist};
    const int widths[3] = {3, 3, histWidth};
    const int k = hist ? 3 : 2;
    if (!strayBlock_) {
        const long long nf = sphk_strays_block_floats(strayCap_, k, widths);
        CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&strayBlock_), sizeof(float) * static_cast<size_t>(nf)));
        CUDA_CALL(cudaMalloc(reinterpret_cast<void**>(&strayGathered_), sizeof(float) * static_cast<size_t>(nf) * boot_.world));
    }
    check(sphk_strays_collect(engine_->ctx(), csF_->addr(), r_.own[0], r_.own[1] - r_.own[0], k, live, widths, strayBlock_, strayCap_),
          "sphk_strays_collect");
    strayPending_ = true;
}

int SlabSPHSystem::straysRouted() {
    if (!strayGathered_) return 0;
    auto* known = dynamic_cast<BasicSPHSolver*>(solver_.get());
    int histWidth = 0;
    const int k = known->historyArray(histWidth) ? 3 : 2;
    const int widths[3] = {3, 3, histWidth};
    std::vector<int> counts(static_cast<size_t>(boot_.world), 0);
    check(sphk_strays_counts(engine_->ctx(), strayGathered_, boot_.world, strayCap_, k, widths, counts.data()), "sphk_strays_counts");
    int total = 0;
    for (const int c : counts) total += c;
    return total;
}

// slabs.SlabSystem._begin_step_native: candidates -> assembled set -> one search -> ranges, counts agreed for the next step
void SlabSPHSystem::beginStep() {
    sphk_ctx* ctx = engine_->ctx();
    auto* known = dynamic_cast<BasicSPHSolver*>(solver_.get());
    int histWidth = 0;
    float* hist = known->historyArray(histWidth);
    const bool L = boot_.rank > 0, R = boot_.rank < boot_.world - 1;
    if (!haveRanges_) {                              // very first step: sort the initial set once, everything local counts as own
        searchAll(nOwn_);
        int b[8];
        readBounds(b);
        if (b[7] != nOwn_) printf("SlabSPHSystem: rank %d: the initial partition left particles outside the local grid\n", boot_.rank);
        r_ = planeRanges(b, w_);
        r_.own[0] = b[0]; r_.own[1] = b[7];
        r_.toLeft[0] = b[0];
        r_.toRight[1] = b[7];
        haveRanges_ = true;
        if (comm_) {
            const int tl[1] = {r_.toLeft[1] - r_.toLeft[0]}, tr[1] = {r_.toRight[1] - r_.toRight[0]};
            int fl[1] = {0}, fr[1] = {0};
            check(sphk_mg_exchange_ints(comm_, tl, tr, fl, fr, 1), "sphk_mg_exchange_ints");
            candFrom_[0] = fl[0]; candFrom_[1] = fr[0];
        }
    }
    const int nl = L ? candFrom_[0] : 0, nr = R ? candFrom_[1] : 0;
    const int own0 = r_.own[0], nOwnPrev = r_.own[1] - r_.own[0];
    int nAll = nl + nOwnPrev + nr;
    if (nAll + (strayPending_ ? boot_.world * strayCap_ : 0) > cap_)
        fail(boot_.rank, "capacity " + std::to_string(cap_) + " exceeded by " + std::to_string(nAll) + " local particles");
    // carried arrays: pos, vel (+ the solver's history array), received straight into their slots of the assembled set
    float* live[3] = {reinterpret_cast<float*>(fluids_->getPosPtr()), reinterpret_cast<float*>(fluids_->getVelPtr()), hist};
    float* alt[3] = {reinterpret_cast<float*>(altPos_->addr()), reinterpret_cast<float*>(altVel_->addr()), altHist_->addr()};
    const int widths[3] = {3, 3, histWidth};
    const int k = hist ? 3 : 2;
    if (comm_) {
        const int sl[2] = {r_.toLeft[0], r_.toLeft[1] - r_.toLeft[0]}, sr[2] = {r_.toRight[0], r_.toRight[1] - r_.toRight[0]};
        const int rl[2] = {0, nl}, rr[2] = {nl + nOwnPrev, nr};
        check(sphk_mg_exchange_slices(comm_, k, live, alt, widths, sl, sr, rl, rr), "sphk_mg_exchange_slices");
    }
    for (int a = 0; a < k; ++a) {
        const size_t wd = static_cast<size_t>(widths[a]);
        check(sphk_copy(ctx, alt[a] + wd * nl, live[a] + wd * own0, static_cast<int>(wd) * nOwnPrev), "sphk_copy");
    }
    if (strayPending_ && comm_) {                   // the strays of every rank, behind the candidates (same order everywhere)
        check(sphk_mg_strays_route(comm_, ctx, strayBlock_, strayGathered_, strayCap_, k, alt, widths, nAll), "sphk_mg_strays_route");
        nAll += boot_.world * strayCap_;
    }
    strayPending_ = false;
    for (int a = 0; a < k; ++a)                      // (DArray pointers are fixed: copy back)
        check(sphk_copy(ctx, live[a], alt[a], widths[a] * nAll), "sphk_copy");
    searchAll(nAll);
    int b[8];
    readBounds(b);
    r_ = planeRanges(b, w_);
    nGhostL_ = r_.ghostL[1] - r_.ghostL[0];
    nOwn_ = r_.own[1] - r_.own[0];
    ownBegin_ = r_.own[0];
    nGhostR_ = r_.ghostR[1] - r_.ghostR[0];
    const int nFirst = r_.first[1] - r_.first[0], nLast = r_.last[1] - r_.last[0];
    if (comm_) {
        // (a) the ordering contract -- my ghost planes must be exactly the neighbours' boundary planes -- checked BEFORE any halo
        // is posted; (b) how many candidates each neighbour will send next step
        const int tl[2] = {nFirst, r_.toLeft[1] - r_.toLeft[0]}, tr[2] = {nLast, r_.toRight[1] - r_.toRight[0]};
        int fl[2] = {0, 0}, fr[2] = {0, 0};
        check(sphk_mg_exchange_ints(comm_, tl, tr, fl, fr, 2), "sphk_mg_exchange_ints");
        if ((L && fl[0] != nGhostL_) || (R && fr[0] != nGhostR_))
            fail(boot_.rank, "ghost planes " + std::to_string(nGhostL_) + "/" + std::to_string(nGhostR_) + " do not match the neighbours' boundary planes " +
                                 std::to_string(fl[0]) + "/" + std::to_string(fr[0]) + " (more strays than SPHK_SLAB_STRAYS in one step?)");
        candFrom_[0] = fl[1]; candFrom_[1] = fr[1];
        int err = 0;
        check(sphk_mg_check(comm_, &err), "sphk_mg_check");
        if (err) fail(boot_.rank, "halo mailbox error bits " + std::to_string(err) + " (see sphk_mg_check)");
    }
    haloRanges_[0] = r_.first[0]; haloRanges_[1] = nFirst; haloRanges_[2] = r_.last[0]; haloRanges_[3] = nLast;
    haloRanges_[4] = r_.ghostL[0]; haloRanges_[5] = nGhostL_; haloRanges_[6] = r_.ghostR[0]; haloRanges_[7] = nGhostR_;
    check(sphk_set_active_range(ctx, r_.own[0], nOwn_), "sphk_set_active_range");
}

float SlabSPHSystem::step() {
    if (!ok_) return 0.0f;
    // implicit viscosity needs a global dot product per CG iteration and a halo of the direction before each product
    const auto* known = dynamic_cast<const BasicSPHSolver*>(solver_.get());
    if (known && known->implicitViscosity() > 0.0f)
        throw std::runtime_error("SlabSPHSystem: implicit viscosity is not supported on slab ranks (single-GPU SPHSystem only)");
    if (known && known->rheologyOn())       // the same solve, plus a shear sweep that would need the ghosts' velocity gradients
        throw std::runtime_error("SlabSPHSystem: non-Newtonian viscosity is not supported on slab ranks (single-GPU SPHSystem only)");
    if (known && known->thermalOn())        // ghosts and strays would need their temperatures carried as a second array
        throw std::runtime_error("SlabSPHSystem: heat transfer is not supported on slab ranks (single-GPU SPHSystem only)");
    if (known && known->adhesionOn())       // the boundary walk and the body reaction are single-context only
        throw std::runtime_error("SlabSPHSystem: adhesion is not supported on slab ranks (single-GPU SPHSystem only)");
    if (known && known->tankForceOn())      // the frame time and the per-step state live in one context
        throw std::runtime_error("SlabSPHSystem: tank motion is not supported on slab ranks (single-GPU SPHSystem only)");
    if (adaptive_)
        throw std::runtime_error("SlabSPHSystem: adaptive time stepping is not supported on slab ranks (single-GPU SPHSystem only)");
    cudaStream_t st = engine_->stream();
    CUDA_CALL(cudaEventRecord(evStart_, st));
    if (strayCap_ > 0 && haveRanges_ && comm_) collectStrays();
    beginStep();
    try {
        solver_->step(fluids_, boundaries_, *csF_, *csB_, spaceSize_, localCellSize_, cellLength_, radius_, dt_, rho0_, rhoB_, stiff_,
                      visc_, G_, surfaceTension_, airPressure_);
    } catch (const char* s) {
        std::cout << s << "\n";
    } catch (...) {
        std::cout << "Unknown Exception at " << __FILE__ << ": line " << __LINE__ << "\n";
    }
    check(sphk_synchronize(engine_->ctx()), "step");
    float milliseconds = 0.0f;
    CUDA_CALL(cudaEventRecord(evStop_, st));
    CUDA_CALL(cudaEventSynchronize(evStop_));
    CUDA_CALL(cudaEventElapsedTime(&milliseconds, evStart_, evStop_));
    return milliseconds;
}
