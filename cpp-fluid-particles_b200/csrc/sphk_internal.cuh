// sphk_internal.cuh -- shared device helpers and the context of libsphk (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "sphk.h"

#define SPHK_EPS (1e-6f)                        // global.h:21
#define SPHK_PI (3.14159265358979323846f)       // global.h:22
#define SPHK_MAX_A (1000.0f)                    // global.h:26
#define SPHK_BLOCK 128
#define SPHK_TILE_CAP 1535                      // records of a tile's staged neighbour windows (+1 dummy slot = 24 KiB per half)
#define SPHK_TILE_WINS 18                       // 9 (dx,dy) rows of the fluid set + 9 of the boundary set
#define SPHK_MAX_BODIES 64                      // kinematic bodies per context (sphk_bodies_init)

// Packed particle records, two 16-byte halves in two arrays (unified index: fluid j < capF, boundary capF + b,
// one far-away zero-mass dummy at capF + capB used as list padding):
//   A[j] = {x, y, z, s}     s = the scalar the NEXT sweep reads from its neighbours: DFSPH stiffness kappa, PBD lambda,
//                           p/rho^2 (pressure force) or |colour gradient|^2 (surface tension).
//                           BOUNDARY records carry their MASS in this slot (their scalar is always 0): a sweep that
//                           gathers only A still has every neighbour's mass (fluid masses are uniform in the
//                           reference's scenes, SPHSystem.cu:73; checked on the device at each search).
//   B[j] = {vx, vy, vz, m}  velocity (0 for boundary particles) and mass
// Sweeps that need position + scalar gather A only (one LDG.128 / one 16-byte slot of a staged tile); sweeps that
// need the velocity gather A and B.  Two arrays (not one 32-byte struct) so that a tile's neighbour windows of A can
// be staged into shared memory by contiguous bulk copies without dragging B along.
struct Rec {
    float4* a; float4* b;
    __host__ __device__ __forceinline__ Rec operator+(long long i) const { return Rec{a + i, b + i}; }
};

// per-launch constants of the smoothing kernels (CUDAFunctions.cuh:23-54,82-98), evaluated once on the host
struct KConst {
    float R;      // support radius
    float hInv;   // 2 / R                 (q = r * hInv)
    float cW;     // 0.25 / (pi R^3)
    float cG;     // 1 / (pi R^5)
    float cLap;   // 45 / (pi R^6)
    float cST;    // 136.0241 / (pi R^9)
    float stOff;  // 0.0156 R^6
    float r2cut;  // R^2 (1 + 1e-5): candidates beyond contribute exactly 0
};

// Device-side iteration control of one adaptive solver loop (DFSPH divergence / density correction): the loop test of
// DFSPHSolver.cu:187,347 evaluated on the device, so that the host enqueues a fixed sequence of launches (max_iter
// iterations, the ones after convergence return at once) instead of reading an error sum back every iteration.
struct LoopState {
    int active;        // the loop condition; kernels of the loop body return immediately when it is 0
    int iters;         // iterations executed
    int minIter, maxIter, reduceFrom;
    float threshold;   // errorThreshold * num * rho0
    float total;       // last error sum (FLT_MAX before the first reduction)
    int pad;
};

// Kinematic rigid bodies (sphk_bodies_*, sphk_search.cu): boundary slots [nStatic, nB) of the PRE-search order belong
// to bodies.  local[] runs parallel to the boundary API arrays (it is permuted with them by every boundary search):
// {r_k (body coordinates), group} with group 0 = the static set, b + 1 = body b.
struct BodyState {
    int nBodies = 0, nStatic = 0, n = 0;   // n: size of the boundary set (static + bodies)
    float* pose = nullptr;           // device [7 * nBodies]: c.xyz, q.xyzw
    float* motion = nullptr;         // device [6 * nBodies]: V.xyz, Omega.xyz (world frame)
    float4* local = nullptr;         // device [capB]
    float4* snapLocal = nullptr;     // device [capB]: pre-sort snapshot of local (the gather permutes out of place)
    float* snapMass = nullptr;       // device [capB]: pre-sort snapshot of the boundary mass
    float* stage = nullptr;          // pinned [6 * SPHK_MAX_BODIES]: staging of sphk_bodies_set_motion
    cudaEvent_t staged = nullptr;    // the copy out of `stage` has been done
    int* decl = nullptr;             // device [capB]: declaration slot of every particle, carried by the search like local[]
    int* snapDecl = nullptr;         // device [capB]: pre-sort snapshot of decl
    int* begin = nullptr;            // device [nBodies + 1]: body_begin of sphk_bodies_init (declaration slots)
    float box[6 * SPHK_MAX_BODIES] = {};   // host: body-frame bounding box of each body's r_k, {lo.xyz, hi.xyz}
    float rmax[SPHK_MAX_BODIES] = {};      // host: max_k |r_k| of each body (the speed bound of sphk_step_speed)
    bool stepped = false;            // sphk_bodies_step has run
    // two-way coupling (sphk_bodies_set_dynamics; DESIGN.md section 2.4)
    float* dyn = nullptr;            // device [SPHK_DYN * nBodies]: M, I.xyz, box lo.xyz, box hi.xyz, clamp box hi.xyz
    double* acc = nullptr;           // device [6 * (n - nStatic)]: {J, H} of every body particle, summed over the step's reactions
    float* impulse = nullptr;        // device [6 * nBodies]: {J, H} of the last integrated step
};
#define SPHK_DYN 16                  // floats per body in BodyState::dyn
__device__ __forceinline__ float body_group(float4 local) { return local.w; }

struct sphk_ctx {
    cudaStream_t stream = nullptr;
    int capF = 0, capB = 0;          // capacities; boundary lives at unified index capF + b
    int3 cs = {0, 0, 0};
    int3 org = {0, 0, 0};            // cell-coordinate origin of the local grid (slab ranks)
    int ncells = 0;
    float cellLength = 0.f;
    int endBit = 32;                 // radix sort key width: ceil(log2(ncells + 1))
    // ---- scratch (device) ----
    int *keys = nullptr, *keysSorted = nullptr, *idx = nullptr, *idxSorted = nullptr;
    void* cubTemp = nullptr; size_t cubTempBytes = 0;
    float4 *snapA = nullptr, *snapB = nullptr;   // [max(capF,capB)] snapshot / Jacobi temp
    Rec rec = {nullptr, nullptr};                // [capF + capB + 1] packed particle records (two 16-byte halves), sorted order
    const void* sTag = nullptr;                  // which caller array rec[].s currently mirrors (nullptr: none)
    float* massRange = nullptr;                  // [2] device: min / max fluid mass of the last search (as float bits)
    float* tmpF = nullptr;                       // [3*capF] permute temp
    float* partial = nullptr;                    // [1024] reduction partials
    LoopState* loops = nullptr;                  // [2] device-side loop control (sphk_loop_*)
    const int* pred = nullptr;                   // non-null: sweeps / reductions run only while *pred != 0
    int* nbr = nullptr;                          // [kmax * capF] neighbour list, nbr[k*capF + i]
    int* cnt = nullptr;                          // [capF] true neighbour count (may exceed kmax)
    float* pinned = nullptr;                     // host pinned scalar
    // ---- state ----
    int nF = 0, nB = 0;
    int actBegin = 0, actCount = -1; // active (owned) range of the sweeps; -1: all
    const int* rangeDev = nullptr;   // non-null: the active range {begin, count} lives in DEVICE memory (slab ranks: computed from
                                     // the cell ranges by sphk_mg_plane_ranges, never read by the host); kernels are launched over
                                     // all nF particles and the ones outside the range return
    int kmax = 96;
    bool useList = true;
    int patch = 0;                   // SPHK_OPT_PATCH (experiment): list sweeps map a block onto a y x z patch of cells
    bool stagedBuild = true;         // build the list from candidate windows staged in shared memory by bulk copies (default);
                                     // false: candidates read from global memory (k_build_list)
    bool simpleBuild = false;        // build the list with the generic cell walk (test reference of k_build_list)
    float skin = 0.f;                // neighbour-list skin as a fraction of R (PBD: positions move inside a step)
    bool listHasSkin = false;        // the current list was built with a skin and displacement is being tracked
    unsigned int* dispMax = nullptr; // device: max squared displacement since the list build (float bits; introspection)
    unsigned char* cellFlag = nullptr; // device [cellFlagCap]: skin lists -- 1 = a particle that moved more than skin/2 since the
    size_t cellFlagCap = 0;            // list build is in this cell or an adjacent one: the particles here walk the cells
    int tile = 0;                    // 1: tile lists -- 16-bit tile-local indices, neighbour windows staged in shared memory by
                                     // bulk copies (k_build_tile / k_sweep_tile); 0: int32 lists gathered from global memory
    int2* tileWin = nullptr;         // [tiles * 18] {first record, count} of the 9 fluid + 9 boundary windows of every tile
    int numSMs = 0;
    unsigned long long searchEpoch = 0, listEpoch = ~0ull;
    int listBegin = 0, listEnd = 0;  // particle range the current list covers
    bool posDirty = false;           // positions changed since the last search
    bool advected = false;           // ... by sphk_advect / sphk_refresh (not only by PBD corrections)
    bool fluidSearched = false, boundarySearched = false, permValid = false;
    const int* lastCsB = nullptr;
    long long launches = 0;
    BodyState* bodies = nullptr;     // non-null after sphk_bodies_init
    float* viscStats = nullptr;      // [2] device: {iterations (int bits), |r|_M / |b|_M} of the last sphk_implicit_viscosity
    // open boundaries (sphk_sinks_apply / sphk_fluid_set_count; allocated on first use)
    int* openDev = nullptr;          // device [2]: {particles the last sphk_sinks_apply removed, sticky check bits}
    int* openPinned = nullptr;       // pinned [1]: the removed count, copied behind the sink kernel
    cudaEvent_t sinkEvent = nullptr; // recorded after that copy
    bool sinksApplied = false;
    mutable bool countSettable = false;   // a fluid search ran and no sweep since (sphk_fluid_set_count is valid)
    // speed bound of adaptive time stepping (sphk_step_speed; allocated on first use)
    unsigned int* speedDev = nullptr;     // device [3]: {fluid max |v|^2, body max bound (float bits), non-finite count}
    unsigned int* speedPinned = nullptr;  // pinned [3]: their copy
    cudaEvent_t speedEvent = nullptr;     // recorded after that copy
};

struct DevScene {
    Rec rec;
    const int* __restrict__ csF;
    const int* __restrict__ csB;
    const int* __restrict__ nbr;
    const int* __restrict__ cnt;
    const float* __restrict__ massRange;
    const unsigned char* cellFlag;   // non-null: skin list in use; a particle whose (current) cell is flagged walks the cells
    int nF, bOff, nbrStride, kmax;
    const int2* tileWin;             // tile lists: the 18 windows of every tile (written by the list builder)
    const int* pred;                 // non-null: the kernel returns at once when *pred == 0 (device-controlled solver loops)
    int dummy;                       // index of a record far away from everything with zero mass: list padding that
                                     // contributes exactly 0 to every particle (group lists cannot pad with "self")
    int iBegin, iEnd;                // sweeps compute particles [iBegin, iEnd)
    const int* rangeDev;             // non-null: ... intersected with the device-resident range {begin, count}
    int patch;                       // > 0: the warps of a block take their 32-particle chunks from 4 runs `patch` chunks apart
    int3 cs, org;
    float cellLength;
    float r2list;                    // candidate cut-off of the cell walk: r2cut, or (R + skin)^2 when building a skin list
    KConst k;
};

__device__ __forceinline__ bool in_range(const DevScene& s, int i) {
    if (s.rangeDev) { const int b = s.rangeDev[0]; return i >= b && i < b + s.rangeDev[1]; }
    return i >= s.iBegin && i < s.iEnd;
}

// ---- tiny float3 algebra (component-wise, left to right) ---------------------------------------
__device__ __forceinline__ float3 f3(float x, float y, float z) { return make_float3(x, y, z); }
__device__ __forceinline__ float3 xyz(float4 v) { return make_float3(v.x, v.y, v.z); }
__device__ __forceinline__ float3 operator+(float3 a, float3 b) { return f3(a.x + b.x, a.y + b.y, a.z + b.z); }
__device__ __forceinline__ float3 operator-(float3 a, float3 b) { return f3(a.x - b.x, a.y - b.y, a.z - b.z); }
__device__ __forceinline__ float3 operator-(float3 a) { return f3(-a.x, -a.y, -a.z); }
__device__ __forceinline__ float3 operator*(float3 a, float s) { return f3(a.x * s, a.y * s, a.z * s); }
__device__ __forceinline__ float3 operator*(float s, float3 a) { return f3(s * a.x, s * a.y, s * a.z); }
__device__ __forceinline__ float3 operator/(float3 a, float s) { return f3(a.x / s, a.y / s, a.z / s); }
__device__ __forceinline__ void operator+=(float3& a, float3 b) { a.x += b.x; a.y += b.y; a.z += b.z; }
__device__ __forceinline__ void operator-=(float3& a, float3 b) { a.x -= b.x; a.y -= b.y; a.z -= b.z; }
__device__ __forceinline__ float dot3(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

__device__ __forceinline__ float3 load3(const float* __restrict__ p, int i) {
    return f3(p[3 * i], p[3 * i + 1], p[3 * i + 2]);
}
__device__ __forceinline__ void store3(float* __restrict__ p, int i, float3 v) {
    p[3 * i] = v.x; p[3 * i + 1] = v.y; p[3 * i + 2] = v.z;
}

// ---- the cell hash, bit-exact with the reference under -use_fast_math ----------------------------
// make_int3(pos / cellLength) compiles to MUFU.RCP + FMUL.FTZ + F2I.FTZ.TRUNC in the reference build
// (CUDAFunctions.cuh:76, src/CMakeLists.txt:43).  div.approx.ftz + cvt.rzi.ftz is that sequence.
__device__ __forceinline__ int cell_coord(float x, float cellLength) {
    float q; int c;
    asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(q) : "f"(x), "f"(cellLength));
    asm("cvt.rzi.ftz.s32.f32 %0, %1;" : "=r"(c) : "f"(q));
    return c;
}
// particlePos2cellIdx, CUDAFunctions.cuh:64-70
__device__ __forceinline__ int cell_index(int x, int y, int z, int3 cs) {
    return (x >= 0 && x < cs.x && y >= 0 && y < cs.y && z >= 0 && z < cs.z) ? ((x * cs.y + y) * cs.z + z)
                                                                            : (cs.x * cs.y * cs.z);
}

// ---- skin lists (PBD: positions move inside a step, PBDSolver.cu:232-256) -------------------------------------------------
// A list built with a skin s holds every pair closer than R(1+s).  It stays complete for two particles that have EACH moved
// less than sR/2 since the build.  A particle that moved further ("fast mover") flags its current cell and the 26 around it:
// every particle that can be within R of it lives in one of those cells, so flagged particles -- the fast mover itself
// included -- fall back to the exact cell walk while everybody else keeps its list.  (Round 1 used the global maximum: one
// splashing particle sent all of them to the cell walk.)
struct SkinTrack {
    const float4* posBuild;      // positions at list build; nullptr: no tracking
    unsigned int* dispMax;       // largest squared displacement seen (introspection only)
    unsigned char* cellFlag;
    float limit2;                // (skin/2 * R)^2
    int3 cs, org;
    float cellLength;
};
__device__ __forceinline__ int cell_coord(float x, float cellLength);
// returns the squared displacement of particle i now at p; flags the neighbourhood of a fast mover
__device__ __forceinline__ float skin_track(const SkinTrack& t, int i, float3 p) {
    const float4 q = t.posBuild[i];
    const float dx = p.x - q.x, dy = p.y - q.y, dz = p.z - q.z;
    const float d2 = dx * dx + dy * dy + dz * dz;
    if (d2 > t.limit2) {
        const int cx = cell_coord(p.x, t.cellLength) - t.org.x, cy = cell_coord(p.y, t.cellLength) - t.org.y,
                  cz = cell_coord(p.z, t.cellLength) - t.org.z;
        for (int x = max(cx - 1, 0); x <= min(cx + 1, t.cs.x - 1); ++x)
            for (int y = max(cy - 1, 0); y <= min(cy + 1, t.cs.y - 1); ++y)
                for (int z = max(cz - 1, 0); z <= min(cz + 1, t.cs.z - 1); ++z)
                    t.cellFlag[(static_cast<size_t>(x) * t.cs.y + y) * t.cs.z + z] = 1;
    }
    return d2;
}
__device__ __forceinline__ void skin_track_max(const SkinTrack& t, float d2) {       // warp-wide; all lanes must call
    for (int o = 16; o > 0; o >>= 1) d2 = fmaxf(d2, __shfl_xor_sync(0xffffffffu, d2, o));
    if ((threadIdx.x & 31) == 0 && __float_as_uint(d2) > *t.dispMax) atomicMax(t.dispMax, __float_as_uint(d2));
}

// ---- record access --------------------------------------------------------------------------------
__device__ __forceinline__ float4 rec_lo(Rec r) { return *r.a; }
__device__ __forceinline__ float4 rec_hi(Rec r) { return *r.b; }
__device__ __forceinline__ void rec_full(Rec r, float4& lo, float4& hi) { lo = *r.a; hi = *r.b; }
__device__ __forceinline__ void rec_store(Rec r, float4 lo, float4 hi) { *r.a = lo; *r.b = hi; }
__device__ __forceinline__ void rec_set_pos(Rec r, float3 p) {
    *reinterpret_cast<float2*>(&r.a->x) = make_float2(p.x, p.y); r.a->z = p.z;
}
__device__ __forceinline__ void rec_set_vel(Rec r, float3 v) {
    *reinterpret_cast<float2*>(&r.b->x) = make_float2(v.x, v.y); r.b->z = v.z;
}
__device__ __forceinline__ void rec_set_s(Rec r, float s) { r.a->w = s; }
__device__ __forceinline__ float rec_m(Rec r) { return r.b->w; }

// ---- smoothing kernels, CUDAFunctions.cuh:23-54,82-98 ------------------------------------------------
// Same functions as the reference, arranged for the issue rate: constants folded per launch (KConst),
// branch-free selects instead of early returns, one MUFU.RCP per gradient.  Differences from the
// reference's expression order are a few ulp per term (<= ~3e-7 relative), far inside the 1e-5 budget.
__device__ __forceinline__ float w_cubic(float r, const KConst& k) {
    const float q = r * k.hInv;
    const float t = 2.0f - q;
    const float w = (q > 1.0f) ? t * t * t : ((3.0f * q - 6.0f) * q * q + 4.0f);
    return (q > 2.0f || q < SPHK_EPS) ? 0.0f : k.cW * w;                   // W(0) = 0: quirk Q1
}
// scalar factor f with grad W = d * f
__device__ __forceinline__ float grad_w_factor(float r, const KConst& k) {
    const float q = r * k.hInv;
    const float p = (q > 1.0f) ? ((12.0f - 3.0f * q) * q - 12.0f) : ((9.0f * q - 12.0f) * q);
    const float f = __fdividef(k.cG, q + SPHK_EPS) * p;
    return (q > 2.0f) ? 0.0f : f;
}
__device__ __forceinline__ float lap_visc(float r, const KConst& k) {
    return (r <= k.R) ? k.cLap * (k.R - r) : 0.0f;
}
// scalar factor f with grad C = d * f (surface-tension kernel gradient; note the reference's -r)
__device__ __forceinline__ float grad_st_factor(float x, const KConst& k) {
    const float e = k.R - x;
    const float e3x3 = (e * e * e) * (x * x * x);
    const float p = (2.0f * x <= k.R) ? (2.0f * e3x3 - k.stOff) : e3x3;
    const float f = -__fdividef(k.cST, x) * p;
    return (x > k.R || x < SPHK_EPS) ? 0.0f : f;
}

#define SPHK_CUDA_TRY(expr)                                  \
    do {                                                     \
        cudaError_t e_ = (expr);                             \
        if (e_ != cudaSuccess) return static_cast<int>(e_);  \
    } while (0)

static inline int sphk_blocks(int n) { return (n + SPHK_BLOCK - 1) / SPHK_BLOCK; }
