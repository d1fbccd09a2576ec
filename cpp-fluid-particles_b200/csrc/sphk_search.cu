// sphk_search.cu -- context lifetime + neighbour search (cell hash -> stable radix sort -> gather ->
// cell ranges) + permutation / element-wise utilities.  Replaces SPHSystem::neighborSearch,
// /root/reference/src/SPHSystem.cu:114-127.
//
// Design (GPU-first, not a translation of the reference's two Thrust sorts with float3 payloads):
//   1. k_hash_snapshot : one pass over pos(+vel): bit-exact cell key (MUFU.RCP path), writes
//                        particle2cell (API, pre-sort order, quirk Q2), the sort key, the identity
//                        index, and a 16-byte-aligned float4 snapshot of pos / vel.
//   2. cub::DeviceRadixSort::SortPairs on (key, index), only ceil(log2(ncells+1)) key bits
//                        -> ONE stable sort of 8-byte pairs instead of two sorts of 16-byte pairs.
//   3. k_gather        : one gather pass writes the sorted API float3 arrays and the packed 32-byte
//                        records {x,y,z,s | vx,vy,vz,m} the sweep kernels gather (one sector per neighbour).
//   4. k_cell_start    : cell_start[c] = lower_bound(sortedKeys, c) -- no atomics, no scan, equals
//                        fill + countingInCell_CUDA + exclusive_scan (SPHSystem.cu:123-125) exactly.
// HBM-bound; algorithmic bytes per particle are listed in DESIGN.md.
#include <cub/device/device_radix_sort.cuh>
#include <algorithm>
#include <cstdio>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>
#include "sphk_internal.cuh"

// kinematic bodies (end of this file)
static void sphk_bodies_release(BodyState* b);
static int sphk_bodies_search(sphk_ctx* c, const sphk_particles* p, int* cell_start);

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(SPHK_BLOCK)
k_hash_snapshot(const float* __restrict__ pos, const float* __restrict__ vel, int n, float cellLength,
                int3 cs, int3 org, int* __restrict__ p2c, int* __restrict__ keys, int* __restrict__ idx,
                float4* __restrict__ snapPos, float4* __restrict__ snapVel) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float3 p = load3(pos, i);
    const int key = cell_index(cell_coord(p.x, cellLength) - org.x, cell_coord(p.y, cellLength) - org.y,
                               cell_coord(p.z, cellLength) - org.z, cs);
    p2c[i] = key;
    keys[i] = key;
    idx[i] = i;
    snapPos[i] = make_float4(p.x, p.y, p.z, 0.f);
    if (vel) { const float3 v = load3(vel, i); snapVel[i] = make_float4(v.x, v.y, v.z, 0.f); }
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_gather(const int* __restrict__ idxSorted, const float4* __restrict__ snapPos,
         const float4* __restrict__ snapVel, const float* __restrict__ mass, int n,
         float* __restrict__ pos, float* __restrict__ vel, Rec rec, int isFluid,
         unsigned int* __restrict__ massRange) {
    const int s = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    float m = 0.f;
    if (s < n) {
        const int src = idxSorted[s];
        float4 p = snapPos[src];
        store3(pos, s, xyz(p));
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (vel) {
            v = snapVel[src];
            store3(vel, s, xyz(v));
            if (!isFluid) v = make_float4(0.f, 0.f, 0.f, 0.f);   // boundary records carry zero velocity / scalar
        }
        m = mass[s];                        // mass is NOT permuted by the reference (Q2): slot s keeps mass[s]
        v.w = m;
        p.w = isFluid ? 0.f : m;            // A.w: neighbour scalar (fluid, none yet) / mass (boundary)
        rec_store(rec + s, p, v);
    }
    if (isFluid) {                          // min / max fluid mass (non-negative floats order like their bits)
        float lo = (s < n) ? m : 3.0e38f, hi = (s < n) ? m : 0.f;
        for (int o = 16; o > 0; o >>= 1) {
            lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if ((threadIdx.x & 31) == 0) {      // almost never taken after the first warps: no atomic storm
            if (__float_as_uint(lo) < massRange[0]) atomicMin(massRange, __float_as_uint(lo));
            if (__float_as_uint(hi) > massRange[1]) atomicMax(massRange + 1, __float_as_uint(hi));
        }
    }
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_cell_start(const int* __restrict__ keysSorted, int n, int ncells, int* __restrict__ cellStart) {
    const int c = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (c > ncells) return;
    int lo = 0, hi = n;                 // first s with keysSorted[s] >= c
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keysSorted[mid] < c) lo = mid + 1; else hi = mid;
    }
    cellStart[c] = lo;
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_permute(const int* __restrict__ idxSorted, const float* __restrict__ src, float* __restrict__ dst,
          int width, int n) {
    const int s = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (s >= n) return;
    const int from = idxSorted[s];
    for (int k = 0; k < width; ++k) dst[s * width + k] = src[from * width + k];
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_repack(const float* __restrict__ pos, const float* __restrict__ vel, const float* __restrict__ mass,
         int n, Rec rec, int isFluid, unsigned int* __restrict__ massRange, const float4* __restrict__ bodyLocal) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    float m = 0.f;
    if (i < n) {
        const float3 p = load3(pos, i);
        m = mass[i];
        float4 v = make_float4(0.f, 0.f, 0.f, m);
        // boundary records with bodies: body particles keep their velocity, the static set keeps zero
        if (vel && (!bodyLocal || body_group(bodyLocal[i]) != 0.f)) { const float3 w = load3(vel, i); v = make_float4(w.x, w.y, w.z, m); }
        rec_store(rec + i, make_float4(p.x, p.y, p.z, isFluid ? 0.f : m), v);
    }
    if (massRange) {
        float lo = (i < n) ? m : 3.0e38f, hi = (i < n) ? m : 0.f;
        for (int o = 16; o > 0; o >>= 1) {
            lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if ((threadIdx.x & 31) == 0) {      // almost never taken after the first warps: no atomic storm
            if (__float_as_uint(lo) < massRange[0]) atomicMin(massRange, __float_as_uint(lo));
            if (__float_as_uint(hi) > massRange[1]) atomicMax(massRange + 1, __float_as_uint(hi));
        }
    }
}

__global__ void k_init_mass_range(unsigned int* r) { r[0] = 0x7f7fffffu; r[1] = 0u; }

__global__ void __launch_bounds__(SPHK_BLOCK) k_fill(float* __restrict__ a, int n, float v) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n) a[i] = v;
}

__global__ void k_rcp(float x, float* out) {
    float one = 1.0f, r;
    asm("div.approx.ftz.f32 %0, %1, %2;" : "=f"(r) : "f"(one), "f"(x));
    // the hash multiplies by MUFU.RCP(x); div.approx(1,x) = 1 * rcp(x) is that value
    *out = r;
}

// abs-sum reduction: fixed-shape two-stage tree (deterministic run to run)
__global__ void __launch_bounds__(256) k_abs_sum_partial(const float* __restrict__ x, int n, float* __restrict__ partial) {
    __shared__ float sm[8];
    float s = 0.f;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) s += fabsf(x[i]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = sm[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) partial[blockIdx.x] = s;
    }
}
__global__ void __launch_bounds__(256) k_abs_sum_final(const float* __restrict__ partial, int m, float* __restrict__ out) {
    __shared__ float sm[8];
    float s = 0.f;
    for (int i = threadIdx.x; i < m; i += 256) s += partial[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = sm[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) *out = s;
    }
}

// ------------------------------------------------------------------------------------------------
template <typename T> static cudaError_t dalloc(T** p, size_t count) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(p), sizeof(T) * (count ? count : 1));
    if (e == cudaSuccess) e = cudaMemset(*p, 0, sizeof(T) * (count ? count : 1));
    return e;
}

extern "C" int sphk_create(sphk_ctx** out, int max_fluid, int max_boundary, const sphk_grid* grid, void* stream) {
    if (!out || !grid || max_fluid <= 0 || max_boundary < 0) return SPHK_ERR_INVALID;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) { cudaGetLastError(); return SPHK_ERR_NO_DEVICE; }
    sphk_ctx* c = new (std::nothrow) sphk_ctx;
    if (!c) return SPHK_ERR_ALLOC;
    c->stream = static_cast<cudaStream_t>(stream);
    c->capF = max_fluid; c->capB = max_boundary;
    c->cs = make_int3(grid->cell_size[0], grid->cell_size[1], grid->cell_size[2]);
    c->org = make_int3(grid->origin[0], grid->origin[1], grid->origin[2]);
    c->ncells = c->cs.x * c->cs.y * c->cs.z;
    c->cellLength = grid->cell_length;
    c->endBit = 1;
    while (c->endBit < 32 && (1ll << c->endBit) <= static_cast<long long>(c->ncells)) ++c->endBit;
    const size_t cap = static_cast<size_t>(max_fluid > max_boundary ? max_fluid : max_boundary);
    const size_t tot = static_cast<size_t>(max_fluid) + static_cast<size_t>(max_boundary);
    cudaError_t e = cudaSuccess;
    if (e == cudaSuccess) e = dalloc(&c->keys, cap);
    if (e == cudaSuccess) e = dalloc(&c->keysSorted, cap);
    if (e == cudaSuccess) e = dalloc(&c->idx, cap);
    if (e == cudaSuccess) e = dalloc(&c->idxSorted, cap);
    if (e == cudaSuccess) e = dalloc(&c->snapA, cap);
    if (e == cudaSuccess) e = dalloc(&c->snapB, cap);
    if (e == cudaSuccess) e = dalloc(&c->rec.a, tot + 1);   // + the far-away zero-mass dummy record (list padding)
    if (e == cudaSuccess) e = dalloc(&c->rec.b, tot + 1);
    if (e == cudaSuccess) {
        const float4 dummy = make_float4(1.0e6f, 1.0e6f, 1.0e6f, 0.f);
        e = cudaMemcpy(c->rec.a + tot, &dummy, sizeof(float4), cudaMemcpyHostToDevice);
    }
    if (e == cudaSuccess) e = dalloc(&c->massRange, 2);
    if (e == cudaSuccess) e = dalloc(&c->dispMax, 1);
    if (e == cudaSuccess) { c->cellFlagCap = static_cast<size_t>(c->ncells) + 1; e = dalloc(&c->cellFlag, c->cellFlagCap); }
    if (e == cudaSuccess) e = dalloc(&c->tmpF, 3 * static_cast<size_t>(max_fluid));
    if (e == cudaSuccess) e = dalloc(&c->partial, 1024);
    if (e == cudaSuccess) e = dalloc(&c->loops, 2);
    if (e == cudaSuccess) e = dalloc(&c->viscStats, 2);
    if (e == cudaSuccess) e = dalloc(&c->rheoStats, 6);
    if (e == cudaSuccess) e = dalloc(&c->heatGroups, SPHK_THERMAL_GROUPS);
    if (e == cudaSuccess) e = dalloc(&c->heatStats, 2);
    if (e == cudaSuccess) e = dalloc(&c->heatRed, 3 * 1024 + 3);
    if (e == cudaSuccess) e = dalloc(&c->adhGroups, SPHK_ADHESION_GROUPS);
    if (e == cudaSuccess) e = dalloc(&c->adhStats, 2);
    if (e == cudaSuccess) e = dalloc(&c->cnt, static_cast<size_t>(max_fluid));
    if (e == cudaSuccess) e = dalloc(&c->tileWin, (static_cast<size_t>(max_fluid) / SPHK_BLOCK + 1) * SPHK_TILE_WINS);
    if (e == cudaSuccess) e = dalloc(&c->chunkAct, static_cast<size_t>(max_fluid) / 32 + 1);
    if (e == cudaSuccess) e = dalloc(&c->chunkStamp, static_cast<size_t>(max_fluid) / 32 + 1);
    if (e == cudaSuccess) e = dalloc(&c->chunkMark, static_cast<size_t>(max_fluid) / 32 + 1);
    if (e == cudaSuccess) {
        int dev = 0;
        cudaGetDevice(&dev);
        e = cudaDeviceGetAttribute(&c->numSMs, cudaDevAttrMultiProcessorCount, dev);
        if (c->numSMs > 256) c->numSMs = 256;
        if (const char* v = std::getenv("SPHK_TILE")) c->tile = v[0] == '1' ? 1 : 0;
    }
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&c->pinned), 64);
    if (e == cudaSuccess) {
        // sized for the widest key any grid can need (32 bits), not only for this grid's: the scratch grows with the number
        // of 8-bit passes, and sphk_set_grid may re-target the context at a grid with more cells without re-allocating
        c->cubTempBytes = 0;
        for (int bits : {c->endBit, 32}) {
            size_t bytes = 0;
            if (e == cudaSuccess) e = cub::DeviceRadixSort::SortPairs(nullptr, bytes, c->keys, c->keysSorted, c->idx, c->idxSorted,
                                                                      static_cast<int>(cap), 0, bits, c->stream);
            if (bytes > c->cubTempBytes) c->cubTempBytes = bytes;
        }
        if (e == cudaSuccess) e = cudaMalloc(&c->cubTemp, c->cubTempBytes ? c->cubTempBytes : 1);
    }
    if (e != cudaSuccess) { sphk_destroy(c); cudaGetLastError(); return e == cudaErrorMemoryAllocation ? SPHK_ERR_ALLOC : static_cast<int>(e); }
    *out = c;
    return SPHK_OK;
}

extern "C" void sphk_destroy(sphk_ctx* c) {
    if (!c) return;
    sphk_checkpoint_release(c);
    cudaFree(c->keys); cudaFree(c->keysSorted); cudaFree(c->idx); cudaFree(c->idxSorted);
    cudaFree(c->snapA); cudaFree(c->snapB); cudaFree(c->rec.a); cudaFree(c->rec.b); cudaFree(c->massRange); cudaFree(c->dispMax); cudaFree(c->cellFlag);
    cudaFree(c->tmpF); cudaFree(c->partial); cudaFree(c->loops); cudaFree(c->viscStats); cudaFree(c->rheoStats); cudaFree(c->heatGroups); cudaFree(c->heatStats); cudaFree(c->heatRed); cudaFree(c->adhGroups); cudaFree(c->adhStats); cudaFree(c->cnt); cudaFree(c->nbr); cudaFree(c->cubTemp); cudaFree(c->tileWin); cudaFree(c->chunkAct); cudaFree(c->chunkStamp); cudaFree(c->chunkMark);
    if (c->pinned) cudaFreeHost(c->pinned);
    if (c->tank) { cudaFree(c->tank->dev); delete c->tank; }
    cudaFree(c->openDev);
    if (c->openPinned) cudaFreeHost(c->openPinned);
    if (c->sinkEvent) cudaEventDestroy(c->sinkEvent);
    cudaFree(c->speedDev);
    if (c->speedPinned) cudaFreeHost(c->speedPinned);
    if (c->speedEvent) cudaEventDestroy(c->speedEvent);
    sphk_bodies_release(c->bodies);
    delete c;
}

extern "C" int sphk_set_option(sphk_ctx* c, int option, int value) {
    if (!c) return SPHK_ERR_INVALID;
    switch (option) {
    case SPHK_OPT_NEIGHBOR_LIST: c->useList = value != 0; return SPHK_OK;
    case SPHK_OPT_LIST_CAPACITY:
        if (value < 8 || value > 1024 || (value & 3)) return SPHK_ERR_INVALID;   // multiple of 4 (int4 batches)
        if (value != c->kmax) {
            if (c->nbr) { cudaStreamSynchronize(c->stream); cudaFree(c->nbr); c->nbr = nullptr; }
            c->kmax = value; c->listEpoch = ~0ull;
        }
        return SPHK_OK;
    case SPHK_OPT_SIMPLE_LIST_BUILD: c->simpleBuild = value != 0; c->listEpoch = ~0ull; return SPHK_OK;
    case SPHK_OPT_PATCH: if (value < 0) return SPHK_ERR_INVALID; c->patch = value; return SPHK_OK;
    case SPHK_OPT_STAGED_LIST_BUILD: c->stagedBuild = value != 0; c->listEpoch = ~0ull; return SPHK_OK;
    case SPHK_OPT_LIST_SKIN:
        if (value < 0 || value > 1000) return SPHK_ERR_INVALID;
        if (value * 0.001f != c->skin) { c->skin = value * 0.001f; c->listEpoch = ~0ull; }
        return SPHK_OK;
    case SPHK_OPT_TILE:
        if (value != 0 && value != 1) return SPHK_ERR_INVALID;
        if (value != c->tile) { c->tile = value; c->listEpoch = ~0ull; }
        return SPHK_OK;
    default: return SPHK_ERR_INVALID;
    }
}

// Re-targets the context at another (sub-)grid of the same cell length: a slab rank whose cuts moved (load re-balancing)
// keeps its context, buffers and lists' storage; both particle sets must be searched again before the next sweep.
extern "C" int sphk_set_grid(sphk_ctx* c, const sphk_grid* grid) {
    if (!c || !grid || grid->cell_size[0] <= 0 || grid->cell_size[1] <= 0 || grid->cell_size[2] <= 0) return SPHK_ERR_INVALID;
    if (grid->cell_length != c->cellLength) return SPHK_ERR_INVALID;
    c->cs = make_int3(grid->cell_size[0], grid->cell_size[1], grid->cell_size[2]);
    c->org = make_int3(grid->origin[0], grid->origin[1], grid->origin[2]);
    c->ncells = c->cs.x * c->cs.y * c->cs.z;
    c->endBit = 1;
    while (c->endBit < 32 && (1ll << c->endBit) <= static_cast<long long>(c->ncells)) ++c->endBit;
    if (static_cast<size_t>(c->ncells) + 1 > c->cellFlagCap) {
        cudaStreamSynchronize(c->stream);
        cudaFree(c->cellFlag);
        c->cellFlag = nullptr;
        c->cellFlagCap = static_cast<size_t>(c->ncells) + 1;
        if (dalloc(&c->cellFlag, c->cellFlagCap) != cudaSuccess) { cudaGetLastError(); c->cellFlagCap = 0; return SPHK_ERR_ALLOC; }
    }
    c->fluidSearched = false; c->boundarySearched = false; c->permValid = false;
    c->listEpoch = ~0ull; c->sTag = nullptr;
    c->actBegin = 0; c->actCount = -1; c->rangeDev = nullptr;
    return SPHK_OK;
}

extern "C" int sphk_synchronize(sphk_ctx* c) {
    if (!c) return SPHK_ERR_INVALID;
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" const char* sphk_error_string(int code) {
    switch (code) {
    case SPHK_OK: return "ok";
    case SPHK_ERR_INVALID: return "sphk: invalid argument";
    case SPHK_ERR_NO_DEVICE: return "sphk: no CUDA device (libsphk has no CPU path)";
    case SPHK_ERR_CAPACITY: return "sphk: particle count exceeds context capacity";
    case SPHK_ERR_STATE: return "sphk: call order violated (neighbour search missing or stale scene)";
    case SPHK_ERR_ALLOC: return "sphk: device allocation failed";
    case SPHK_ERR_COMM: return "sphk: multi-GPU exchange failed (NCCL unavailable / error, or mailbox wiring missing)";
    default: return code > 0 ? cudaGetErrorString(static_cast<cudaError_t>(code)) : "sphk: unknown error";
    }
}

extern "C" long long sphk_launch_count(const sphk_ctx* c) { return c ? c->launches : 0; }
extern "C" int sphk_add_launches(sphk_ctx* c, long long n) { if (!c) return SPHK_ERR_INVALID; c->launches += n; return SPHK_OK; }

extern "C" int sphk_device_rcp(sphk_ctx* c, float x, float* out_host) {
    if (!c || !out_host) return SPHK_ERR_INVALID;
    k_rcp<<<1, 1, 0, c->stream>>>(x, c->partial);
    c->launches++;
    SPHK_CUDA_TRY(cudaMemcpyAsync(c->pinned, c->partial, sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    *out_host = *c->pinned;
    return SPHK_OK;
}

// ------------------------------------------------------------------------------------------------
extern "C" int sphk_neighbor_search(sphk_ctx* c, int which, const sphk_particles* p, int* cell_start) {
    if (!c || !p || !cell_start || !p->pos || !p->mass || !p->particle2cell || p->n <= 0) return SPHK_ERR_INVALID;
    const bool fluid = which == 0;
    if (fluid && !p->vel) return SPHK_ERR_INVALID;
    const int n = p->n;
    if (n > (fluid ? c->capF : c->capB)) return SPHK_ERR_CAPACITY;
    if (!fluid && c->bodies) return sphk_bodies_search(c, p, cell_start);   // carries mass and body frame along
    const int off = fluid ? 0 : c->capF;
    cudaStream_t st = c->stream;
    k_hash_snapshot<<<sphk_blocks(n), SPHK_BLOCK, 0, st>>>(p->pos, p->vel, n, c->cellLength, c->cs, c->org, p->particle2cell,
                                                          c->keys, c->idx, c->snapA, c->snapB);
    size_t tb = c->cubTempBytes;
    SPHK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cubTemp, tb, c->keys, c->keysSorted, c->idx, c->idxSorted, n, 0,
                                                  c->endBit, st));
    if (fluid) k_init_mass_range<<<1, 1, 0, st>>>(reinterpret_cast<unsigned int*>(c->massRange));
    k_gather<<<sphk_blocks(n), SPHK_BLOCK, 0, st>>>(c->idxSorted, c->snapA, c->snapB, p->mass, n, p->pos, p->vel,
                                                   c->rec + off, fluid ? 1 : 0, reinterpret_cast<unsigned int*>(c->massRange));
    k_cell_start<<<sphk_blocks(c->ncells + 1), SPHK_BLOCK, 0, st>>>(c->keysSorted, n, c->ncells, cell_start);
    c->launches += 3 + 4;   // 3 own kernels + CUB onesweep (histogram, scan, <=3 passes): counted as 4
    if (fluid) { c->nF = n; c->fluidSearched = true; c->permValid = true; c->searchEpoch++; c->posDirty = false; c->advected = false; c->sTag = nullptr;
                 c->actBegin = 0; c->actCount = -1; c->countSettable = true; }
    else { c->nB = n; c->boundarySearched = true; c->listEpoch = ~0ull; c->permValid = false; }
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_permute(sphk_ctx* c, float* array, int width, int n) {
    if (!c || !array || (width != 1 && width != 3)) return SPHK_ERR_INVALID;
    if (!c->permValid || n != c->nF) return SPHK_ERR_STATE;
    if (array == c->sTag) c->sTag = nullptr;
    k_permute<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(c->idxSorted, array, c->tmpF, width, n);
    c->launches++;
    SPHK_CUDA_TRY(cudaMemcpyAsync(array, c->tmpF, sizeof(float) * static_cast<size_t>(n) * width,
                                  cudaMemcpyDeviceToDevice, c->stream));
    return SPHK_OK;
}

extern "C" int sphk_refresh(sphk_ctx* c, const sphk_scene* s) {
    if (!c || !s) return SPHK_ERR_INVALID;
    if (!c->fluidSearched || s->fluid.n != c->nF) return SPHK_ERR_STATE;
    k_init_mass_range<<<1, 1, 0, c->stream>>>(reinterpret_cast<unsigned int*>(c->massRange));
    k_repack<<<sphk_blocks(c->nF), SPHK_BLOCK, 0, c->stream>>>(s->fluid.pos, s->fluid.vel, s->fluid.mass, c->nF, c->rec, 1,
                                                              reinterpret_cast<unsigned int*>(c->massRange), nullptr);
    c->launches++;
    c->posDirty = true;
    c->advected = true;
    c->sTag = nullptr;
    if (c->boundarySearched && s->boundary.pos && s->boundary.n == c->nB) {
        const float4* local = c->bodies ? c->bodies->local : nullptr;
        k_repack<<<sphk_blocks(c->nB), SPHK_BLOCK, 0, c->stream>>>(s->boundary.pos, local ? s->boundary.vel : nullptr,
                                                                  s->boundary.mass, c->nB, c->rec + c->capF, 0, nullptr, local);
        c->launches++;
    }
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_axpy(float* __restrict__ pos, const float* __restrict__ vel, int n3, float dt) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i < n3) pos[i] = pos[i] + dt * vel[i];
}

extern "C" int sphk_particles_advect(float* pos, const float* vel, int n, float dt, void* stream) {
    if (!pos || !vel || n < 0) return SPHK_ERR_INVALID;
    if (n == 0) return SPHK_OK;
    k_axpy<<<sphk_blocks(3 * n), SPHK_BLOCK, 0, static_cast<cudaStream_t>(stream)>>>(pos, vel, 3 * n, dt);
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_fill(sphk_ctx* c, float* array, int n, float value) {
    if (!c || !array || n < 0) return SPHK_ERR_INVALID;
    if (n == 0) return SPHK_OK;
    if (array == c->sTag) c->sTag = nullptr;
    k_fill<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(array, n, value);
    c->launches++;
    // A fill of an API mass array AFTER the search that packed it (the reference kernels read mass[] live) is not
    // mirrored here: the next sphk_neighbor_search / sphk_refresh re-packs it.  SPHSystem's constructor fills the
    // fluid mass before the fluid search that precedes its first sweep (SPHSystem.cu:73-76), so the class layer never
    // needs the refresh.
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_copy(sphk_ctx* c, float* dst, const float* src, int n_floats) {
    if (!c || !dst || !src || n_floats < 0) return SPHK_ERR_INVALID;
    if (dst == c->sTag) c->sTag = nullptr;
    // a copy is no launch (act_mark() does not see it): one into an array of the DFSPH error sweeps ends their reuse
    if (dst == c->tok.density || dst == c->tok.alpha || dst == c->tok.error || dst == c->tok.stiff) c->tok.kind = 0;
    // ... and one over the velocities of the last correct sweep ends their epoch
    if (c->velArr && dst < c->velArr + 3 * static_cast<size_t>(c->capF) && dst + n_floats > c->velArr) c->velMark = -1;
    SPHK_CUDA_TRY(cudaMemcpyAsync(dst, src, sizeof(float) * static_cast<size_t>(n_floats), cudaMemcpyDeviceToDevice, c->stream));
    return SPHK_OK;
}

extern "C" int sphk_reduce_abs_sum(sphk_ctx* c, const float* x, int n, float* host_out) {
    if (!c || !x || !host_out || n < 0) return SPHK_ERR_INVALID;
    int blocks = (n + 256 * 8 - 1) / (256 * 8);
    if (blocks < 1) blocks = 1;
    if (blocks > 1024) blocks = 1024;
    k_abs_sum_partial<<<blocks, 256, 0, c->stream>>>(x, n, c->partial);
    k_abs_sum_final<<<1, 256, 0, c->stream>>>(c->partial, blocks, c->partial);
    c->launches += 2; c->credited += 2; c->velCredited += 2;   // writes only the partials
    SPHK_CUDA_TRY(cudaMemcpyAsync(c->pinned, c->partial, sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    *host_out = *c->pinned;
    return SPHK_OK;
}

// ---- device-side scene generation (SURVEY 8f-4): initSPHSystem(), main.cpp:73-116, without a host-side particle array ---------
// The fluid block in the reference's push order (i = y outermost, j = x, k = z innermost; main.cpp:76-85), optionally
// restricted to the x-columns [jBegin, jBegin + jCount) (a slab rank generates only its own columns; the restriction keeps
// the relative order, which is all the stable sort sees).  Arithmetic as the host code performs it: float multiply, then
// float add, no contraction -- the positions are bit-identical to scene.py / main.cpp.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_scene_fluid_block(float* __restrict__ pos, int nz, int jBegin, int jCount, long long count, float ox, float oy, float oz, float spacing) {
    const long long p = static_cast<long long>(blockIdx.x) * SPHK_BLOCK + threadIdx.x;
    if (p >= count) return;
    const int k = static_cast<int>(p % nz);
    const long long q = p / nz;
    const int j = jBegin + static_cast<int>(q % jCount);
    const int i = static_cast<int>(q / jCount);
    pos[3 * p] = __fadd_rn(ox, __fmul_rn(spacing, static_cast<float>(j)));
    pos[3 * p + 1] = __fadd_rn(oy, __fmul_rn(spacing, static_cast<float>(i)));
    pos[3 * p + 2] = __fadd_rn(oz, __fmul_rn(spacing, static_cast<float>(k)));
}

extern "C" int sphk_scene_fluid_block(float* pos_out, int nx, int ny, int nz, const float origin[3], float spacing, int j_begin,
                                      int j_count, void* stream) {
    if (!pos_out || !origin || nx <= 0 || ny <= 0 || nz <= 0 || j_begin < 0 || j_count < 0 || j_begin + j_count > nx) return SPHK_ERR_INVALID;
    const long long count = static_cast<long long>(ny) * j_count * nz;
    if (count == 0) return SPHK_OK;
    const long long blocks = (count + SPHK_BLOCK - 1) / SPHK_BLOCK;
    if (blocks > 0x7fffffffLL) return SPHK_ERR_INVALID;
    k_scene_fluid_block<<<static_cast<unsigned int>(blocks), SPHK_BLOCK, 0, static_cast<cudaStream_t>(stream)>>>(
        pos_out, nz, j_begin, j_count, count, origin[0], origin[1], origin[2], spacing);
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// The six-face boundary shell, main.cpp:89-116: lattice c = 2 * cellSize per axis, point (i,j,k) -> 0.99 * ((i,j,k) / (c - 1) *
// spaceSize) + 0.005 * spaceSize, pushed as front/back pairs (i in cx, j in cy), top/bottom pairs (i in cx, j in cz - 2),
// left/right pairs (i in cy - 2, j in cz - 2).  IEEE divide / multiply / add, no contraction.
__device__ __forceinline__ float shell_coord(int idx, int c, float space) {
    const float x = __fmul_rn(__fdiv_rn(static_cast<float>(idx), static_cast<float>(c - 1)), space);
    return __fadd_rn(__fmul_rn(0.99f, x), __fmul_rn(0.005f, space));
}
__global__ void __launch_bounds__(SPHK_BLOCK)
k_scene_boundary_shell(float* __restrict__ pos, int cx, int cy, int cz, float sx, float sy, float sz, long long n0, long long n1, long long n2) {
    const long long p = static_cast<long long>(blockIdx.x) * SPHK_BLOCK + threadIdx.x;
    if (p >= n0 + n1 + n2) return;
    int ix, iy, iz;
    if (p < n0) {                       // front and back
        const long long q = p >> 1; const int second = static_cast<int>(p & 1);
        ix = static_cast<int>(q / cy); iy = static_cast<int>(q % cy); iz = second ? cz - 1 : 0;
    } else if (p < n0 + n1) {           // top and bottom
        const long long r = p - n0, q = r >> 1; const int second = static_cast<int>(r & 1);
        ix = static_cast<int>(q / (cz - 2)); iz = static_cast<int>(q % (cz - 2)) + 1; iy = second ? cy - 1 : 0;
    } else {                            // left and right
        const long long r = p - n0 - n1, q = r >> 1; const int second = static_cast<int>(r & 1);
        iy = static_cast<int>(q / (cz - 2)) + 1; iz = static_cast<int>(q % (cz - 2)) + 1; ix = second ? cx - 1 : 0;
    }
    pos[3 * p] = shell_coord(ix, cx, sx);
    pos[3 * p + 1] = shell_coord(iy, cy, sy);
    pos[3 * p + 2] = shell_coord(iz, cz, sz);
}

extern "C" long long sphk_scene_boundary_count(const int cell_size[3]) {
    if (!cell_size) return -1;
    const long long cx = 2LL * cell_size[0], cy = 2LL * cell_size[1], cz = 2LL * cell_size[2];
    if (cx < 2 || cy < 2 || cz < 2) return -1;
    return 2 * cx * cy + 2 * cx * (cz - 2) + 2 * (cy - 2) * (cz - 2);
}

extern "C" int sphk_scene_boundary_shell(float* pos_out, const int cell_size[3], const float space[3], void* stream) {
    if (!pos_out || !cell_size || !space) return SPHK_ERR_INVALID;
    const long long total = sphk_scene_boundary_count(cell_size);
    if (total <= 0) return SPHK_ERR_INVALID;
    const int cx = 2 * cell_size[0], cy = 2 * cell_size[1], cz = 2 * cell_size[2];
    const long long n0 = 2LL * cx * cy, n1 = 2LL * cx * (cz - 2), n2 = 2LL * (cy - 2) * (cz - 2);
    const long long blocks = (total + SPHK_BLOCK - 1) / SPHK_BLOCK;
    k_scene_boundary_shell<<<static_cast<unsigned int>(blocks), SPHK_BLOCK, 0, static_cast<cudaStream_t>(stream)>>>(
        pos_out, cx, cy, cz, space[0], space[1], space[2], n0, n1, n2);
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

// ---- device-side loop control (adaptive DFSPH, DFSPHSolver.cu:187,205-207,347,360) ----------------------------------
__global__ void k_loop_begin(LoopState* st, int minIter, int maxIter, float threshold, int reduceFrom) {
    st->iters = 0; st->minIter = minIter; st->maxIter = maxIter; st->reduceFrom = reduceFrom;
    st->threshold = threshold; st->total = 3.402823466e38f;
    st->active = ((0 < minIter) || (st->total > threshold)) && (0 < maxIter) ? 1 : 0;
}
// first stage of the error sum of iteration iters + 1 (same fixed-shape tree as sphk_reduce_abs_sum: same sum, bit for bit)
__global__ void __launch_bounds__(256) k_loop_partial(const LoopState* st, const float* __restrict__ x, int n, float* __restrict__ partial) {
    if (!st->active || st->iters + 1 < st->reduceFrom) return;
    __shared__ float sm[8];
    float s = 0.f;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < n; i += gridDim.x * 256) s += fabsf(x[i]);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 8) {
        s = sm[threadIdx.x];
        for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
        if (threadIdx.x == 0) partial[blockIdx.x] = s;
    }
}
// second stage + the loop test: ++iter; total = sum (from iteration reduceFrom on); active = (iter < min || total > thr) && iter < max
__global__ void __launch_bounds__(256) k_loop_finish(LoopState* st, const float* __restrict__ partial, int m) {
    if (!st->active) return;
    __shared__ float sm[8];
    const int iters = st->iters + 1;
    float total = st->total;
    if (iters >= st->reduceFrom) {
        float s = 0.f;
        for (int i = threadIdx.x; i < m; i += 256) s += partial[i];
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x < 8) {
            s = sm[threadIdx.x];
            for (int o = 4; o > 0; o >>= 1) s += __shfl_xor_sync(0xffu, s, o);
            if (threadIdx.x == 0) sm[0] = s;
        }
        __syncthreads();
        total = sm[0];
    }
    if (threadIdx.x == 0) {
        st->iters = iters;
        st->total = total;
        st->active = ((iters < st->minIter) || (total > st->threshold)) && (iters < st->maxIter) ? 1 : 0;
    }
}

extern "C" int sphk_loop_begin(sphk_ctx* c, int slot, int min_iter, int max_iter, float threshold, int reduce_from_iter) {
    if (!c || slot < 0 || slot > 1 || max_iter < 0) return SPHK_ERR_INVALID;
    k_loop_begin<<<1, 1, 0, c->stream>>>(c->loops + slot, min_iter, max_iter, threshold, reduce_from_iter);
    c->launches++; c->credited++; c->velCredited++;   // loop control writes only its LoopState (chunk activity stays valid)
    c->pred = &c->loops[slot].active;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_loop_next(sphk_ctx* c, int slot, const float* error, int n) {
    if (!c || slot < 0 || slot > 1 || !error || n < 0) return SPHK_ERR_INVALID;
    int blocks = (n + 256 * 8 - 1) / (256 * 8);
    if (blocks < 1) blocks = 1;
    if (blocks > 1024) blocks = 1024;
    k_loop_partial<<<blocks, 256, 0, c->stream>>>(c->loops + slot, error, n, c->partial);
    k_loop_finish<<<1, 256, 0, c->stream>>>(c->loops + slot, c->partial, blocks);
    c->launches += 2; c->credited += 2; c->velCredited += 2;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_loop_end(sphk_ctx* c, int slot) {
    if (!c || slot < 0 || slot > 1) return SPHK_ERR_INVALID;
    c->pred = nullptr;
    return SPHK_OK;
}

extern "C" int sphk_loop_iterations(sphk_ctx* c, int slot, int* iterations_host, float* last_total_host) {
    if (!c || slot < 0 || slot > 1 || !iterations_host) return SPHK_ERR_INVALID;
    LoopState h;
    SPHK_CUDA_TRY(cudaMemcpyAsync(&h, c->loops + slot, sizeof(h), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    *iterations_host = h.iters;
    if (last_total_host) *last_total_host = h.total;
    return SPHK_OK;
}

// generate_dots_CUDA, vbo.cu:26-44
__global__ void __launch_bounds__(SPHK_BLOCK)
k_export_dots(const float* __restrict__ pos, const float* __restrict__ density, float* __restrict__ dot, float* __restrict__ color, int n) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    store3(dot, i, load3(pos, i));
    const float d = density[i];
    const float3 blue = f3(0.34f, 0.46f, 0.7f), white = f3(0.9f, 0.9f, 0.9f), pink = f3(1.0f, 0.4f, 0.7f);
    float3 c;
    if (d < 0.75f) c = blue;
    else if (d < 1.0f) { const float w = (d - 0.75f) * 4.0f; c = w * white + (1 - w) * blue; }
    else { float w = (powf(d, 2) - 1.0f) * 4.0f; w = fminf(w, 1.0f); c = (1 - w) * white + w * pink; }
    store3(color, i, c);
}

extern "C" int sphk_export_dots(sphk_ctx* c, const sphk_particles* p, float* dot, float* color) {
    if (!c || !p || !p->pos || !p->density || !dot || !color || p->n < 0) return SPHK_ERR_INVALID;
    if (p->n > 0) k_export_dots<<<sphk_blocks(p->n), SPHK_BLOCK, 0, c->stream>>>(p->pos, p->density, dot, color, p->n);
    c->launches++;
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_get_permutation(sphk_ctx* c, int* perm_out, int n) {
    if (!c || !perm_out) return SPHK_ERR_INVALID;
    if (!c->permValid || n != c->nF) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaMemcpyAsync(perm_out, c->idxSorted, sizeof(int) * static_cast<size_t>(n), cudaMemcpyDeviceToDevice, c->stream));
    return SPHK_OK;
}

// ---- kinematic rigid bodies (no reference counterpart; DESIGN.md section 2.3) ------------------------------------------
// A body is a rigid set of boundary particles given in body coordinates r_k, with pose {c, q} and motion {V, Omega} (world
// frame) in device memory.  Per step (sphk_bodies_step, before the fluid search):
//   c <- c + dt V;  q <- normalize(dq (x) q), dq = (sin(|Omega| dt / 2) Omega / |Omega|, cos(|Omega| dt / 2))
//   x_k = c + R(q) r_k,  v_k = V + Omega x (x_k - c)
// then the boundary set is searched again.  Every boundary search of a context with bodies carries the mass and the
// {r_k, group} of each particle with it (the reference leaves boundary masses in place, Q2: they are computed once, after
// the one search) and keeps the body velocities in the records; the static set keeps v = 0.

__device__ void pose_rotate(float* P, double wx, double wy, double wz, double w, float dt);

// R(q) as a row-major 3x3 matrix in double
__device__ void quat_matrix(const float* q, double R[9]) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    R[0] = 1.0 - 2.0 * (y * y + z * z); R[1] = 2.0 * (x * y - z * w);       R[2] = 2.0 * (x * z + y * w);
    R[3] = 2.0 * (x * y + z * w);       R[4] = 1.0 - 2.0 * (x * x + z * z); R[5] = 2.0 * (y * z - x * w);
    R[6] = 2.0 * (x * z - y * w);       R[7] = 2.0 * (y * z + x * w);       R[8] = 1.0 - 2.0 * (x * x + y * y);
}

// Wall contact of a dynamic body (DESIGN.md section 2.4): the 8 corners of its body-frame bounding box at the new pose must lie
// in the box the fluid is clamped to, [0, 0.99 space] per axis.  The centre moves back by the largest penetration of each axis
// and the outward component of V is zeroed (inelastic, frictionless; no torque).
__device__ void body_contact(float* P, float* V, const float* D) {
    double R[9];
    quat_matrix(P + 3, R);
    double lo[3] = {1e300, 1e300, 1e300}, hi[3] = {-1e300, -1e300, -1e300};
    for (int k = 0; k < 8; ++k) {
        const double r[3] = {D[(k & 1) ? 7 : 4], D[(k & 2) ? 8 : 5], D[(k & 4) ? 9 : 6]};
        for (int a = 0; a < 3; ++a) {
            const double x = P[a] + R[3 * a] * r[0] + R[3 * a + 1] * r[1] + R[3 * a + 2] * r[2];
            lo[a] = fmin(lo[a], x); hi[a] = fmax(hi[a], x);
        }
    }
    for (int a = 0; a < 3; ++a) {
        if (lo[a] < 0.0) {
            P[a] = static_cast<float>(P[a] - lo[a]);
            V[a] = fmaxf(V[a], 0.f);
        } else if (hi[a] > D[10 + a]) {
            P[a] = static_cast<float>(P[a] - (hi[a] - D[10 + a]));
            V[a] = fminf(V[a], 0.f);
        }
    }
}

// One thread per body.  The update is evaluated in double from the float pose and rounded once: with -use_fast_math the
// float sin / cos would be the approximate intrinsics.  dyn (sphk_bodies_set_dynamics, else null): dynamic bodies then
// meet the walls.
__global__ void k_bodies_pose(float* __restrict__ pose, float* __restrict__ motion, int nBodies, float dt,
                              const float* __restrict__ dyn) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nBodies) return;
    float* P = pose + 7 * b;
    float* M = motion + 6 * b;
    for (int a = 0; a < 3; ++a) P[a] = __fadd_rn(P[a], __fmul_rn(dt, M[a]));
    const double wx = M[3], wy = M[4], wz = M[5];
    const double w = sqrt(wx * wx + wy * wy + wz * wz);
    if (w != 0.0) pose_rotate(P, wx, wy, wz, w, dt);        // dq = identity otherwise: q stays bit for bit
    if (dyn && dyn[SPHK_DYN * b] > 0.f) body_contact(P, M, dyn + SPHK_DYN * b);
}

// q <- normalize(dq (x) q) of k_bodies_pose
__device__ void pose_rotate(float* P, double wx, double wy, double wz, double w, float dt) {
    const double h = 0.5 * w * static_cast<double>(dt), s = sin(h) / w;
    const double dx = s * wx, dy = s * wy, dz = s * wz, dw = cos(h);
    const double qx = P[3], qy = P[4], qz = P[5], qw = P[6];
    // Hamilton product dq (x) q: (dw qv + qw dv + dv x qv, dw qw - dv . qv)
    double rx = dw * qx + qw * dx + (dy * qz - dz * qy);
    double ry = dw * qy + qw * dy + (dz * qx - dx * qz);
    double rz = dw * qz + qw * dz + (dx * qy - dy * qx);
    double rw = dw * qw - (dx * qx + dy * qy + dz * qz);
    const double inv = 1.0 / sqrt(rx * rx + ry * ry + rz * rz + rw * rw);
    P[3] = static_cast<float>(rx * inv); P[4] = static_cast<float>(ry * inv);
    P[5] = static_cast<float>(rz * inv); P[6] = static_cast<float>(rw * inv);
}

// Places the body particles at their pose (pos and vel of the boundary API arrays; static particles are left alone) and
// snapshots mass and {r_k, group} for the gather, which permutes them out of place.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_bodies_place(const float4* __restrict__ local, const float* __restrict__ pose, const float* __restrict__ motion,
               const float* __restrict__ mass, int n, float* __restrict__ pos, float* __restrict__ vel,
               float4* __restrict__ snapLocal, float* __restrict__ snapMass, const int* __restrict__ decl,
               int* __restrict__ snapDecl) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float4 l = local[i];
    snapLocal[i] = l;
    snapMass[i] = mass[i];
    snapDecl[i] = decl[i];
    const int g = static_cast<int>(body_group(l));
    if (g == 0) return;
    const float* P = pose + 7 * (g - 1);
    const float* M = motion + 6 * (g - 1);
    const float3 c = f3(P[0], P[1], P[2]), qv = f3(P[3], P[4], P[5]), r = xyz(l);
    const float qw = P[6];
    // R(q) r = r + qw t + qv x t, t = 2 qv x r (exactly r for the identity)
    const float3 t = f3(2.f * (qv.y * r.z - qv.z * r.y), 2.f * (qv.z * r.x - qv.x * r.z), 2.f * (qv.x * r.y - qv.y * r.x));
    const float3 rr = f3(r.x + qw * t.x + (qv.y * t.z - qv.z * t.y), r.y + qw * t.y + (qv.z * t.x - qv.x * t.z),
                         r.z + qw * t.z + (qv.x * t.y - qv.y * t.x));
    const float3 x = c + rr;
    const float3 d = x - c, W = f3(M[3], M[4], M[5]);
    const float3 v = f3(M[0] + (W.y * d.z - W.z * d.y), M[1] + (W.z * d.x - W.x * d.z), M[2] + (W.x * d.y - W.y * d.x));
    store3(pos, i, x);
    store3(vel, i, v);
}

// The boundary gather of a context with bodies: sorted pos / vel, mass and {r_k, group} permuted along, records with the
// body velocities (static records: v = 0)
__global__ void __launch_bounds__(SPHK_BLOCK)
k_bodies_gather(const int* __restrict__ idxSorted, const float4* __restrict__ snapPos, const float4* __restrict__ snapVel,
                const float* __restrict__ snapMass, const float4* __restrict__ snapLocal, int n, float* __restrict__ pos,
                float* __restrict__ vel, float* __restrict__ mass, float4* __restrict__ local, Rec rec,
                const int* __restrict__ snapDecl, int* __restrict__ decl) {
    const int s = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (s >= n) return;
    const int src = idxSorted[s];
    float4 p = snapPos[src], v = snapVel[src];
    const float4 l = snapLocal[src];
    const float m = snapMass[src];
    store3(pos, s, xyz(p));
    store3(vel, s, xyz(v));
    mass[s] = m;
    local[s] = l;
    decl[s] = snapDecl[src];
    if (body_group(l) == 0.f) v = make_float4(0.f, 0.f, 0.f, 0.f);
    v.w = m;
    p.w = m;
    rec_store(rec + s, p, v);
}

// End of step of every body (DESIGN.md section 2.4), one block per body.  The block sums the {J, H} its particles gathered over
// the step's reactions in a fixed shape (strided partials, then a tree; deterministic) and clears them.  Thread 0 reports
// them and, for a dynamic body (M > 0), updates the motion in double, rounded once:
//   V += J / M + dt G;  L = R diag(I) R^T Omega + H;  Omega = R diag(1/I) R^T L   (R from the current pose)
#define SPHK_INTEGRATE_THREADS 256
__global__ void __launch_bounds__(SPHK_INTEGRATE_THREADS)
k_bodies_integrate(const int* __restrict__ begin, int nStatic, double* __restrict__ acc, const float* __restrict__ pose,
                   float* __restrict__ motion, const float* __restrict__ dyn, float* __restrict__ impulse, float dt, float3 G,
                   const float* __restrict__ tankG) {
    __shared__ double red[6][SPHK_INTEGRATE_THREADS];
    const int b = blockIdx.x, t = threadIdx.x;
    const int k0 = begin[b] - nStatic, k1 = begin[b + 1] - nStatic;
    double s[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int k = k0 + t; k < k1; k += SPHK_INTEGRATE_THREADS)
        for (int q = 0; q < 6; ++q) { s[q] += acc[6 * static_cast<size_t>(k) + q]; acc[6 * static_cast<size_t>(k) + q] = 0.0; }
    for (int q = 0; q < 6; ++q) red[q][t] = s[q];
    __syncthreads();
    for (int w = SPHK_INTEGRATE_THREADS / 2; w > 0; w >>= 1) {
        if (t < w)
            for (int q = 0; q < 6; ++q) red[q][t] += red[q][t + w];
        __syncthreads();
    }
    if (t != 0) return;
    const double J[3] = {red[0][0], red[1][0], red[2][0]}, H[3] = {red[3][0], red[4][0], red[5][0]};
    for (int q = 0; q < 3; ++q) { impulse[6 * b + q] = static_cast<float>(J[q]); impulse[6 * b + 3 + q] = static_cast<float>(H[q]); }
    const float* D = dyn + SPHK_DYN * b;
    const double M = D[0];
    if (!(M > 0.0)) return;                                  // held: kinematic, the reaction is only reported
    float* Mo = motion + 6 * b;
    const double g[3] = {tankG ? tankG[0] : G.x, tankG ? tankG[1] : G.y, tankG ? tankG[2] : G.z};   // tank motion: R (G - a_w)
    for (int a = 0; a < 3; ++a) Mo[a] = static_cast<float>(Mo[a] + J[a] / M + static_cast<double>(dt) * g[a]);
    double R[9];
    quat_matrix(pose + 7 * b + 3, R);
    const double I[3] = {D[1], D[2], D[3]}, W[3] = {Mo[3], Mo[4], Mo[5]};
    double wb[3], L[3], lb[3];
    for (int a = 0; a < 3; ++a) wb[a] = R[a] * W[0] + R[3 + a] * W[1] + R[6 + a] * W[2];              // R^T Omega
    for (int a = 0; a < 3; ++a) L[a] = R[3 * a] * I[0] * wb[0] + R[3 * a + 1] * I[1] * wb[1] + R[3 * a + 2] * I[2] * wb[2] + H[a];
    for (int a = 0; a < 3; ++a) lb[a] = (R[a] * L[0] + R[3 + a] * L[1] + R[6 + a] * L[2]) / I[a];    // diag(1/I) R^T L
    for (int a = 0; a < 3; ++a) Mo[3 + a] = static_cast<float>(R[3 * a] * lb[0] + R[3 * a + 1] * lb[1] + R[3 * a + 2] * lb[2]);
}

static void sphk_bodies_release(BodyState* b) {
    if (!b) return;
    cudaFree(b->pose); cudaFree(b->motion); cudaFree(b->local); cudaFree(b->snapLocal); cudaFree(b->snapMass);
    cudaFree(b->decl); cudaFree(b->snapDecl); cudaFree(b->begin); cudaFree(b->dyn); cudaFree(b->acc); cudaFree(b->impulse);
    if (b->stage) cudaFreeHost(b->stage);
    if (b->staged) cudaEventDestroy(b->staged);
    delete b;
}

static int sphk_bodies_search(sphk_ctx* c, const sphk_particles* p, int* cell_start) {
    BodyState* B = c->bodies;
    const int n = p->n;
    if (!p->vel || n != B->n) return SPHK_ERR_INVALID;      // the set declared by sphk_bodies_init
    cudaStream_t st = c->stream;
    k_bodies_place<<<sphk_blocks(n), SPHK_BLOCK, 0, st>>>(B->local, B->pose, B->motion, p->mass, n, p->pos, p->vel,
                                                         B->snapLocal, B->snapMass, B->decl, B->snapDecl);
    k_hash_snapshot<<<sphk_blocks(n), SPHK_BLOCK, 0, st>>>(p->pos, p->vel, n, c->cellLength, c->cs, c->org, p->particle2cell,
                                                          c->keys, c->idx, c->snapA, c->snapB);
    size_t tb = c->cubTempBytes;
    SPHK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(c->cubTemp, tb, c->keys, c->keysSorted, c->idx, c->idxSorted, n, 0,
                                                  c->endBit, st));
    k_bodies_gather<<<sphk_blocks(n), SPHK_BLOCK, 0, st>>>(c->idxSorted, c->snapA, c->snapB, B->snapMass, B->snapLocal, n,
                                                          p->pos, p->vel, p->mass, B->local, c->rec + c->capF, B->snapDecl,
                                                          B->decl);
    k_cell_start<<<sphk_blocks(c->ncells + 1), SPHK_BLOCK, 0, st>>>(c->keysSorted, n, c->ncells, cell_start);
    c->launches += 4 + 4;
    c->nB = n; c->boundarySearched = true; c->listEpoch = ~0ull; c->permValid = false;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

static bool all_finite(const float* x, int n) {
    for (int i = 0; i < n; ++i)
        if (!(x[i] - x[i] == 0.f)) return false;
    return true;
}

extern "C" int sphk_bodies_init(sphk_ctx* c, const sphk_particles* boundary, int n_static, int n_bodies, const int* body_begin,
                                const float* local_xyz, const float* pose, const float* motion) {
    if (!c || !boundary || !boundary->pos || !boundary->vel || !boundary->mass || !body_begin || !local_xyz || !pose || !motion)
        return SPHK_ERR_INVALID;
    const int n = boundary->n;
    if (n_bodies < 1 || n_bodies > SPHK_MAX_BODIES || n_static < 0 || n > c->capB || body_begin[0] != n_static ||
        body_begin[n_bodies] != n)
        return SPHK_ERR_INVALID;
    for (int b = 0; b < n_bodies; ++b)
        if (body_begin[b + 1] < body_begin[b]) return SPHK_ERR_INVALID;
    if (!all_finite(pose, 7 * n_bodies) || !all_finite(motion, 6 * n_bodies) || !all_finite(local_xyz, 3 * (n - n_static)))
        return SPHK_ERR_INVALID;
    if (c->bodies || c->boundarySearched) return SPHK_ERR_STATE;   // bodies are declared before the first boundary search
    std::vector<float4> local(static_cast<size_t>(n), make_float4(0.f, 0.f, 0.f, 0.f));
    for (int b = 0; b < n_bodies; ++b)
        for (int k = body_begin[b]; k < body_begin[b + 1]; ++k) {
            const float* r = local_xyz + 3 * static_cast<size_t>(k - n_static);
            local[k] = make_float4(r[0], r[1], r[2], static_cast<float>(b + 1));
        }
    std::vector<float> q(pose, pose + 7 * n_bodies);
    for (int b = 0; b < n_bodies; ++b) {                     // unit quaternions (a zero one is refused)
        float* Q = q.data() + 7 * b + 3;
        const double l = std::sqrt(double(Q[0]) * Q[0] + double(Q[1]) * Q[1] + double(Q[2]) * Q[2] + double(Q[3]) * Q[3]);
        if (!(l > 0.0)) return SPHK_ERR_INVALID;
        if (l != 1.0)
            for (int a = 0; a < 4; ++a) Q[a] = static_cast<float>(Q[a] / l);
    }
    BodyState* B = new (std::nothrow) BodyState;
    if (!B) return SPHK_ERR_ALLOC;
    B->nBodies = n_bodies; B->nStatic = n_static; B->n = n;
    for (int b = 0; b < n_bodies; ++b) {                     // body-frame bounding boxes (wall contact of dynamic bodies)
        float* box = B->box + 6 * b;
        for (int a = 0; a < 3; ++a) { box[a] = 0.f; box[3 + a] = 0.f; }
        for (int k = body_begin[b]; k < body_begin[b + 1]; ++k)
            for (int a = 0; a < 3; ++a) {
                const float r = local_xyz[3 * static_cast<size_t>(k - n_static) + a];
                if (k == body_begin[b] || r < box[a]) box[a] = r;
                if (k == body_begin[b] || r > box[3 + a]) box[3 + a] = r;
            }
        double r2 = 0.0;
        for (int k = body_begin[b]; k < body_begin[b + 1]; ++k) {
            const float* r = local_xyz + 3 * static_cast<size_t>(k - n_static);
            r2 = std::fmax(r2, double(r[0]) * r[0] + double(r[1]) * r[1] + double(r[2]) * r[2]);
        }
        B->rmax[b] = static_cast<float>(std::sqrt(r2));
    }
    std::vector<int> decl(static_cast<size_t>(n));
    for (int k = 0; k < n; ++k) decl[k] = k;
    const size_t cap = static_cast<size_t>(c->capB);
    cudaError_t e = dalloc(&B->pose, 7 * static_cast<size_t>(n_bodies));
    if (e == cudaSuccess) e = dalloc(&B->motion, 6 * static_cast<size_t>(n_bodies));
    if (e == cudaSuccess) e = dalloc(&B->local, cap);
    if (e == cudaSuccess) e = dalloc(&B->snapLocal, cap);
    if (e == cudaSuccess) e = dalloc(&B->snapMass, cap);
    if (e == cudaSuccess) e = dalloc(&B->decl, cap);
    if (e == cudaSuccess) e = dalloc(&B->snapDecl, cap);
    if (e == cudaSuccess) e = dalloc(&B->begin, static_cast<size_t>(n_bodies) + 1);
    if (e == cudaSuccess) e = cudaMemcpy(B->decl, decl.data(), sizeof(int) * decl.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(B->begin, body_begin, sizeof(int) * (n_bodies + 1), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&B->stage), sizeof(float) * 6 * SPHK_MAX_BODIES);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&B->staged, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMemcpy(B->pose, q.data(), sizeof(float) * q.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(B->motion, motion, sizeof(float) * 6 * n_bodies, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(B->local, local.data(), sizeof(float4) * local.size(), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaEventRecord(B->staged, c->stream);
    if (e != cudaSuccess) { sphk_bodies_release(B); cudaGetLastError(); return e == cudaErrorMemoryAllocation ? SPHK_ERR_ALLOC : static_cast<int>(e); }
    c->bodies = B;
    return SPHK_OK;
}

extern "C" int sphk_bodies_set_motion(sphk_ctx* c, const float* motion_host) {
    if (!c || !motion_host) return SPHK_ERR_INVALID;
    if (!c->bodies) return SPHK_ERR_STATE;
    BodyState* B = c->bodies;
    if (!all_finite(motion_host, 6 * B->nBodies)) return SPHK_ERR_INVALID;
    // the staging buffer is reused: wait until the copy of the previous change has left it (a no-op once the stream got there)
    SPHK_CUDA_TRY(cudaEventSynchronize(B->staged));
    std::memcpy(B->stage, motion_host, sizeof(float) * 6 * B->nBodies);
    SPHK_CUDA_TRY(cudaMemcpyAsync(B->motion, B->stage, sizeof(float) * 6 * B->nBodies, cudaMemcpyHostToDevice, c->stream));
    SPHK_CUDA_TRY(cudaEventRecord(B->staged, c->stream));
    return SPHK_OK;
}

extern "C" int sphk_bodies_step(sphk_ctx* c, const sphk_particles* boundary, int* cell_start_boundary, float dt) {
    if (!c || !boundary || !cell_start_boundary || !boundary->pos || !boundary->vel || !boundary->mass || !boundary->particle2cell)
        return SPHK_ERR_INVALID;
    if (!(dt > 0.f) || !all_finite(&dt, 1)) return SPHK_ERR_INVALID;
    if (!c->bodies || !c->boundarySearched) return SPHK_ERR_STATE;
    if (boundary->n != c->nB) return SPHK_ERR_STATE;
    BodyState* B = c->bodies;
    k_bodies_pose<<<1, SPHK_MAX_BODIES, 0, c->stream>>>(B->pose, B->motion, B->nBodies, dt, B->dyn);
    c->launches++;
    B->stepped = true;
    return sphk_bodies_search(c, boundary, cell_start_boundary);
}

extern "C" int sphk_bodies_set_dynamics(sphk_ctx* c, const float* mass_inertia, const float space[3]) {
    if (!c || !mass_inertia || !space) return SPHK_ERR_INVALID;
    if (!c->bodies) return SPHK_ERR_STATE;
    BodyState* B = c->bodies;
    if (!all_finite(mass_inertia, 4 * B->nBodies) || !all_finite(space, 3)) return SPHK_ERR_INVALID;
    for (int a = 0; a < 3; ++a)
        if (!(space[a] > 0.f)) return SPHK_ERR_INVALID;
    for (int b = 0; b < B->nBodies; ++b) {
        const float* m = mass_inertia + 4 * b;
        if (!(m[0] >= 0.f) || m[1] < 0.f || m[2] < 0.f || m[3] < 0.f) return SPHK_ERR_INVALID;
        if (m[0] > 0.f && !(m[1] > 0.f && m[2] > 0.f && m[3] > 0.f)) return SPHK_ERR_INVALID;
    }
    if (B->dyn || B->stepped) return SPHK_ERR_STATE;        // once, before the first sphk_bodies_step
    bool anyDynamic = false;
    for (int b = 0; b < B->nBodies; ++b) anyDynamic = anyDynamic || mass_inertia[4 * b] > 0.f;
    if (anyDynamic && c->tank && c->tank->on && c->tank->rotates) return SPHK_ERR_STATE;   // no rigid dynamics in a rotating frame
    std::vector<float> dyn(static_cast<size_t>(SPHK_DYN) * B->nBodies, 0.f);
    for (int b = 0; b < B->nBodies; ++b) {
        float* D = dyn.data() + SPHK_DYN * b;
        for (int a = 0; a < 4; ++a) D[a] = mass_inertia[4 * b + a];
        for (int a = 0; a < 6; ++a) D[4 + a] = B->box[6 * b + a];
        for (int a = 0; a < 3; ++a) D[10 + a] = space[a] * .99f;     // the fluid's clamp box (k_advect's clamp_axis)
    }
    const size_t nk = static_cast<size_t>(B->n - B->nStatic);
    cudaError_t e = dalloc(&B->dyn, dyn.size());
    if (e == cudaSuccess) e = dalloc(&B->acc, 6 * nk);
    if (e == cudaSuccess) e = dalloc(&B->impulse, 6 * static_cast<size_t>(B->nBodies));
    if (e == cudaSuccess) e = cudaMemcpy(B->dyn, dyn.data(), sizeof(float) * dyn.size(), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(B->dyn); cudaFree(B->acc); cudaFree(B->impulse);
        B->dyn = nullptr; B->acc = nullptr; B->impulse = nullptr;
        cudaGetLastError();
        return e == cudaErrorMemoryAllocation ? SPHK_ERR_ALLOC : static_cast<int>(e);
    }
    B->anyDynamic = anyDynamic;
    return SPHK_OK;
}

extern "C" int sphk_bodies_integrate(sphk_ctx* c, float dt, const float G[3]) {
    if (!c || !G) return SPHK_ERR_INVALID;
    if (!(dt > 0.f) || !all_finite(&dt, 1) || !all_finite(G, 3)) return SPHK_ERR_INVALID;
    if (!c->bodies || !c->bodies->dyn) return SPHK_ERR_STATE;
    const BodyState* B = c->bodies;
    k_bodies_integrate<<<B->nBodies, SPHK_INTEGRATE_THREADS, 0, c->stream>>>(B->begin, B->nStatic, B->acc, B->pose, B->motion,
                                                                             B->dyn, B->impulse, dt, make_float3(G[0], G[1], G[2]),
                                                                             c->tank && c->tank->on ? c->tank->dev->state + 3 : nullptr);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_bodies_set_body_motion(sphk_ctx* c, int body, const float motion[6]) {
    if (!c || !motion) return SPHK_ERR_INVALID;
    if (!c->bodies) return SPHK_ERR_STATE;
    BodyState* B = c->bodies;
    if (body < 0 || body >= B->nBodies || !all_finite(motion, 6)) return SPHK_ERR_INVALID;
    SPHK_CUDA_TRY(cudaEventSynchronize(B->staged));         // the staging buffer is shared with sphk_bodies_set_motion
    std::memcpy(B->stage + 6 * body, motion, sizeof(float) * 6);
    SPHK_CUDA_TRY(cudaMemcpyAsync(B->motion + 6 * body, B->stage + 6 * body, sizeof(float) * 6, cudaMemcpyHostToDevice, c->stream));
    SPHK_CUDA_TRY(cudaEventRecord(B->staged, c->stream));
    return SPHK_OK;
}

extern "C" int sphk_bodies_get_motion(sphk_ctx* c, float* motion_host) {
    if (!c || !motion_host) return SPHK_ERR_INVALID;
    if (!c->bodies) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaMemcpyAsync(motion_host, c->bodies->motion, sizeof(float) * 6 * c->bodies->nBodies, cudaMemcpyDeviceToHost,
                                  c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SPHK_OK;
}

extern "C" int sphk_bodies_get_impulse(sphk_ctx* c, float* impulse_host) {
    if (!c || !impulse_host) return SPHK_ERR_INVALID;
    if (!c->bodies || !c->bodies->dyn) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaMemcpyAsync(impulse_host, c->bodies->impulse, sizeof(float) * 6 * c->bodies->nBodies, cudaMemcpyDeviceToHost,
                                  c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SPHK_OK;
}

extern "C" int sphk_bodies_get_pose(sphk_ctx* c, float* pose_host) {
    if (!c || !pose_host) return SPHK_ERR_INVALID;
    if (!c->bodies) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaMemcpyAsync(pose_host, c->bodies->pose, sizeof(float) * 7 * c->bodies->nBodies, cudaMemcpyDeviceToHost,
                                  c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SPHK_OK;
}

extern "C" int sphk_bodies_get_local(sphk_ctx* c, float* local_out) {
    if (!c || !local_out) return SPHK_ERR_INVALID;
    if (!c->bodies || !c->boundarySearched) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaMemcpyAsync(local_out, c->bodies->local, sizeof(float4) * static_cast<size_t>(c->nB), cudaMemcpyDeviceToDevice,
                                  c->stream));
    return SPHK_OK;
}

// ---- open boundaries: emitters and sinks (no reference counterpart; DESIGN.md section 2.6) ----------------------------------
// A step of a system with emitters or sinks: k_open_sinks_mark over the n live slots, k_open_emit into [n, n + e), the
// unchanged fluid search over n + e slots (marked particles get the out-of-grid key and sort behind the live ones), then
// sphk_fluid_set_count(L = n + e - removed) with k_open_count_check.  The schedule of an emitter lives on the host
// (sphk_emitter_advance); the kernels only write what it decided.

#define SPHK_EMIT_LAYERS 32          // layer offsets per emission launch (kernel parameters: no host-to-device copy)
struct EmitLayers { float delta[SPHK_EMIT_LAYERS]; };
struct SinkBoxes { float b[6 * SPHK_MAX_SINKS]; };

// One thread per emitted particle k W H + b W + a of the launch's layers; float operations in the order of sphk.h, no contraction.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_open_emit(float* __restrict__ pos, float* __restrict__ vel, float* __restrict__ mass, float* __restrict__ density,
            float* __restrict__ pressure, float* __restrict__ hist, int histKind, int dst, int W, int H, int nLayers, EmitLayers L,
            float3 o, float3 d, float3 e1, float3 e2, float s, float u, float m0, float dt) {
    const int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    const int per = W * H;
    if (t >= nLayers * per) return;
    const int k = t / per, r = t - k * per, b = r / W, a = r - b * W;
    const float ta = __fmul_rn(__fsub_rn(static_cast<float>(a), __fmul_rn(0.5f, static_cast<float>(W - 1))), s);
    const float tb = __fmul_rn(__fsub_rn(static_cast<float>(b), __fmul_rn(0.5f, static_cast<float>(H - 1))), s);
    const float delta = L.delta[k];
    const float3 x = f3(__fadd_rn(__fadd_rn(__fadd_rn(o.x, __fmul_rn(ta, e1.x)), __fmul_rn(tb, e2.x)), __fmul_rn(delta, d.x)),
                        __fadd_rn(__fadd_rn(__fadd_rn(o.y, __fmul_rn(ta, e1.y)), __fmul_rn(tb, e2.y)), __fmul_rn(delta, d.y)),
                        __fadd_rn(__fadd_rn(__fadd_rn(o.z, __fmul_rn(ta, e1.z)), __fmul_rn(tb, e2.z)), __fmul_rn(delta, d.z)));
    const float3 v = f3(__fmul_rn(u, d.x), __fmul_rn(u, d.y), __fmul_rn(u, d.z));
    const int i = dst + t;
    store3(pos, i, x);
    store3(vel, i, v);
    mass[i] = m0;
    density[i] = 0.f;
    pressure[i] = 0.f;
    if (histKind == 1) hist[i] = 0.f;
    else if (histKind == 2)
        store3(hist, i, f3(__fsub_rn(x.x, __fmul_rn(dt, v.x)), __fsub_rn(x.y, __fmul_rn(dt, v.y)), __fsub_rn(x.z, __fmul_rn(dt, v.z))));
}

// Marks the live particles inside a sink (lo <= x < hi on all axes) and counts them: one ballot per warp, one integer add per
// warp with a hit (order-independent, so the count is deterministic).  Every lane reaches the ballot.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_open_sinks_mark(float* __restrict__ pos, float* __restrict__ vel, int n, SinkBoxes B, int nBoxes, int* __restrict__ count) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    bool in = false;
    if (i < n) {
        const float3 p = load3(pos, i);
        for (int k = 0; k < nBoxes; ++k) {
            const float* q = B.b + 6 * k;
            in = in || (p.x >= q[0] && p.x < q[3] && p.y >= q[1] && p.y < q[4] && p.z >= q[2] && p.z < q[5]);
        }
        if (in) {
            store3(pos, i, f3(-1.0e6f, -1.0e6f, -1.0e6f));
            store3(vel, i, f3(0.f, 0.f, 0.f));
        }
    }
    const unsigned int hits = __ballot_sync(0xffffffffu, in);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(count, __popc(hits));
}

// After the search of n + e slots: the in-grid particles must be exactly the L live ones
__global__ void k_open_count_check(const int* __restrict__ cellStart, int ncells, int L, int* __restrict__ bits) {
    if (cellStart[ncells] != L) atomicOr(bits, 1);
}

static bool open_range_active(const sphk_ctx* c) { return c->actCount >= 0 || c->rangeDev != nullptr; }

static int open_alloc(sphk_ctx* c) {
    if (c->openDev) return SPHK_OK;
    cudaError_t e = dalloc(&c->openDev, 2);
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&c->openPinned), sizeof(int));
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->sinkEvent, cudaEventDisableTiming);
    if (e != cudaSuccess) {
        cudaFree(c->openDev); c->openDev = nullptr;
        if (c->openPinned) cudaFreeHost(c->openPinned);
        c->openPinned = nullptr;
        if (c->sinkEvent) cudaEventDestroy(c->sinkEvent);
        c->sinkEvent = nullptr;
        cudaGetLastError();
        return e == cudaErrorMemoryAllocation ? SPHK_ERR_ALLOC : static_cast<int>(e);
    }
    return SPHK_OK;
}

// {d, e1, e2} in double (sphk.h): d normalised; e1 = normalize(d x y^), or normalize(d x x^) when |d . y^| > 0.9; e2 = e1 x d
static int emitter_axes(const sphk_emitter* e, double d[3], double e1[3], double e2[3]) {
    if (!e) return SPHK_ERR_INVALID;
    if (!all_finite(e->origin, 3) || !all_finite(e->direction, 3) || !all_finite(&e->speed, 1) || !all_finite(&e->spacing, 1))
        return SPHK_ERR_INVALID;
    if (!(e->speed > 0.f) || !(e->spacing > 0.f) || e->width < 1 || e->height < 1) return SPHK_ERR_INVALID;
    const double l = std::sqrt(double(e->direction[0]) * e->direction[0] + double(e->direction[1]) * e->direction[1] +
                               double(e->direction[2]) * e->direction[2]);
    if (!(l > 0.0)) return SPHK_ERR_INVALID;
    for (int a = 0; a < 3; ++a) d[a] = e->direction[a] / l;
    double c[3];
    if (std::fabs(d[1]) > 0.9) { c[0] = 0.0; c[1] = d[2]; c[2] = -d[1]; }   // d x x^
    else { c[0] = -d[2]; c[1] = 0.0; c[2] = d[0]; }                           // d x y^
    const double lc = std::sqrt(c[0] * c[0] + c[1] * c[1] + c[2] * c[2]);
    for (int a = 0; a < 3; ++a) e1[a] = c[a] / lc;
    e2[0] = e1[1] * d[2] - e1[2] * d[1];
    e2[1] = e1[2] * d[0] - e1[0] * d[2];
    e2[2] = e1[0] * d[1] - e1[1] * d[0];
    return SPHK_OK;
}

extern "C" int sphk_emitter_axes(const sphk_emitter* e, float axes_out[9]) {
    if (!axes_out) return SPHK_ERR_INVALID;
    double d[3], e1[3], e2[3];
    const int rc = emitter_axes(e, d, e1, e2);
    if (rc != SPHK_OK) return rc;
    for (int a = 0; a < 3; ++a) {
        axes_out[a] = static_cast<float>(d[a]);
        axes_out[3 + a] = static_cast<float>(e1[a]);
        axes_out[6 + a] = static_cast<float>(e2[a]);
    }
    return SPHK_OK;
}

extern "C" int sphk_emitter_advance(const sphk_emitter* e, double* carry, float dt, int max_layers, float* offsets_out,
                                    int* scheduled_out) {
    double d[3], e1[3], e2[3];
    if (emitter_axes(e, d, e1, e2) != SPHK_OK || !carry || !scheduled_out || max_layers < 0 || (max_layers > 0 && !offsets_out))
        return SPHK_ERR_INVALID;
    if (!(dt >= 0.f) || !all_finite(&dt, 1) || !(*carry >= 0.0) || !std::isfinite(*carry)) return SPHK_ERR_INVALID;
    const double s = e->spacing;
    double c = *carry + static_cast<double>(e->speed) * static_cast<double>(dt);
    if (c / s > 65536.0) return SPHK_ERR_INVALID;
    int k = 0;
    while (c >= s && k <= 65536) {
        const double delta = c - s;
        if (k < max_layers) offsets_out[k] = static_cast<float>(delta);
        c -= s;
        ++k;
    }
    *carry = c;
    *scheduled_out = k;
    return SPHK_OK;
}

extern "C" int sphk_emit(sphk_ctx* c, const sphk_particles* fluid, int dst_begin, const sphk_emitter* e, int n_layers,
                         const float* offsets_host, float m0, float dt, float* history, int history_kind) {
    if (!c || !fluid || !fluid->pos || !fluid->vel || !fluid->mass || !fluid->density || !fluid->pressure) return SPHK_ERR_INVALID;
    double d[3], e1[3], e2[3];
    if (emitter_axes(e, d, e1, e2) != SPHK_OK || n_layers < 0 || dst_begin < 0 || (n_layers > 0 && !offsets_host)) return SPHK_ERR_INVALID;
    if (!(m0 > 0.f) || !all_finite(&m0, 1) || !(dt >= 0.f) || !all_finite(&dt, 1)) return SPHK_ERR_INVALID;
    if (history_kind < 0 || history_kind > 2 || (history_kind != 0 && !history)) return SPHK_ERR_INVALID;
    if (n_layers > 0 && !all_finite(offsets_host, n_layers)) return SPHK_ERR_INVALID;
    if (open_range_active(c)) return SPHK_ERR_STATE;
    const long long per = static_cast<long long>(e->width) * e->height;
    if (dst_begin + per * n_layers > c->capF) return SPHK_ERR_CAPACITY;
    if (n_layers == 0) return SPHK_OK;
    float ax[9];
    sphk_emitter_axes(e, ax);
    const float3 o = make_float3(e->origin[0], e->origin[1], e->origin[2]);
    const float3 dv = make_float3(ax[0], ax[1], ax[2]), a1 = make_float3(ax[3], ax[4], ax[5]), a2 = make_float3(ax[6], ax[7], ax[8]);
    for (int k0 = 0; k0 < n_layers; k0 += SPHK_EMIT_LAYERS) {
        const int nl = std::min(SPHK_EMIT_LAYERS, n_layers - k0);
        EmitLayers L{};
        for (int k = 0; k < nl; ++k) L.delta[k] = offsets_host[k0 + k];
        const int count = static_cast<int>(per * nl);
        k_open_emit<<<sphk_blocks(count), SPHK_BLOCK, 0, c->stream>>>(fluid->pos, fluid->vel, fluid->mass, fluid->density, fluid->pressure,
                                                                     history, history_kind, dst_begin + static_cast<int>(per * k0),
                                                                     e->width, e->height, nl, L, o, dv, a1, a2, e->spacing, e->speed, m0, dt);
        c->launches++;
    }
    c->fluidSearched = false; c->permValid = false;     // the new slots reach the records through the next fluid search
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_sinks_apply(sphk_ctx* c, const sphk_particles* fluid, const float* boxes_host, int n_boxes) {
    if (!c || !fluid || !fluid->pos || !fluid->vel || fluid->n < 0 || n_boxes < 0 || n_boxes > SPHK_MAX_SINKS) return SPHK_ERR_INVALID;
    if (n_boxes > 0 && (!boxes_host || !all_finite(boxes_host, 6 * n_boxes))) return SPHK_ERR_INVALID;
    for (int k = 0; k < n_boxes; ++k)
        for (int a = 0; a < 3; ++a)
            if (!(boxes_host[6 * k + a] < boxes_host[6 * k + 3 + a])) return SPHK_ERR_INVALID;
    if (open_range_active(c)) return SPHK_ERR_STATE;
    if (fluid->n > c->capF) return SPHK_ERR_CAPACITY;
    const int rc = open_alloc(c);
    if (rc != SPHK_OK) return rc;
    SinkBoxes B{};
    for (int k = 0; k < 6 * n_boxes; ++k) B.b[k] = boxes_host[k];
    SPHK_CUDA_TRY(cudaMemsetAsync(c->openDev, 0, sizeof(int), c->stream));
    if (fluid->n > 0) {
        k_open_sinks_mark<<<sphk_blocks(fluid->n), SPHK_BLOCK, 0, c->stream>>>(fluid->pos, fluid->vel, fluid->n, B, n_boxes, c->openDev);
        c->launches++;
    }
    SPHK_CUDA_TRY(cudaMemcpyAsync(c->openPinned, c->openDev, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaEventRecord(c->sinkEvent, c->stream));
    c->sinksApplied = true;
    c->fluidSearched = false; c->permValid = false;     // marked positions reach the records through the next fluid search
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_sinks_removed(sphk_ctx* c, int* removed_host) {
    if (!c || !removed_host) return SPHK_ERR_INVALID;
    if (!c->sinksApplied) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaEventSynchronize(c->sinkEvent));
    *removed_host = *c->openPinned;
    return SPHK_OK;
}

extern "C" int sphk_fluid_set_count(sphk_ctx* c, const int* cell_start_fluid, int L) {
    if (!c || !cell_start_fluid || L < 0) return SPHK_ERR_INVALID;
    if (open_range_active(c) || !c->fluidSearched || !c->countSettable || L > c->nF) return SPHK_ERR_STATE;
    const int rc = open_alloc(c);
    if (rc != SPHK_OK) return rc;
    k_open_count_check<<<1, 1, 0, c->stream>>>(cell_start_fluid, c->ncells, L, c->openDev + 1);
    c->launches++;
    c->nF = L;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_open_check(sphk_ctx* c, int* error_bits_host) {
    if (!c || !error_bits_host) return SPHK_ERR_INVALID;
    int bits = 0;
    if (c->openDev) {
        SPHK_CUDA_TRY(cudaMemcpyAsync(&bits, c->openDev + 1, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    *error_bits_host = bits;
    return SPHK_OK;
}

// ---- CFL-adaptive time stepping (no reference counterpart; DESIGN.md section 2.8) ---------------------------------------------
// The rule lives on the host (sphk_time_step); the device only measures the speed bound the rule starts from.

struct BodyRadii { float r[SPHK_MAX_BODIES]; };

__device__ __forceinline__ bool finite_bits(float x) { return (__float_as_uint(x) & 0x7f800000u) != 0x7f800000u; }

// out[0] = max |v|^2 over the finite fluid velocities, out[1] = max |V| + |Omega| r_max over the finite body motions (block 0),
// out[2] += the particles and bodies left out.  The maxima are non-negative floats, so their bits order as unsigned integers: one
// atomicMax per block gives the same bits whatever order the blocks run in.  Every lane of a block reaches every shuffle and ballot.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_step_speed(const float* __restrict__ vel, int n, const float* __restrict__ motion, int nBodies, BodyRadii R,
             unsigned int* __restrict__ out) {
    __shared__ unsigned int warpMax[SPHK_BLOCK / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned int m = 0u;
    for (int i = blockIdx.x * SPHK_BLOCK + threadIdx.x; i - static_cast<int>(threadIdx.x) < n; i += gridDim.x * SPHK_BLOCK) {
        bool bad = false;
        if (i < n) {
            const float3 v = load3(vel, i);
            bad = !(finite_bits(v.x) && finite_bits(v.y) && finite_bits(v.z));
            if (!bad) m = max(m, __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y)), __fmul_rn(v.z, v.z))));
        }
        const unsigned int hits = __ballot_sync(0xffffffffu, bad);
        if (lane == 0 && hits) atomicAdd(out + 2, static_cast<unsigned int>(__popc(hits)));
    }
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) warpMax[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < SPHK_BLOCK / 32; ++w) m = max(m, warpMax[w]);
        if (m) atomicMax(out, m);
    }
    if (blockIdx.x == 0 && threadIdx.x < nBodies) {
        const float* M = motion + 6 * threadIdx.x;
        bool ok = true;
        for (int a = 0; a < 6; ++a) ok = ok && finite_bits(M[a]);
        if (!ok) {
            atomicAdd(out + 2, 1u);
        } else {
            const float v = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[0], M[0]), __fmul_rn(M[1], M[1])), __fmul_rn(M[2], M[2])));
            const float w = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(M[3], M[3]), __fmul_rn(M[4], M[4])), __fmul_rn(M[5], M[5])));
            const float b = __fadd_rn(v, __fmul_rn(w, R.r[threadIdx.x]));
            if (finite_bits(b)) atomicMax(out + 1, __float_as_uint(b));
            else atomicAdd(out + 2, 1u);
        }
    }
}

static bool rule_valid(const sphk_time_step_rule* r) {
    const double f[5] = {r->cfl, r->dt_min, r->dt_max, r->radius, r->gravity};
    for (double x : f)
        if (!std::isfinite(x)) return false;
    return r->cfl > 0.0 && r->dt_min > 0.0 && r->dt_min <= r->dt_max && r->radius > 0.0 && r->gravity >= 0.0;
}

extern "C" int sphk_time_step(const sphk_time_step_rule* r, double v_max, double dt_prev, double remaining, float* dt_out,
                              int* flags_out) {
    if (!r || !dt_out || !flags_out || !rule_valid(r)) return SPHK_ERR_INVALID;
    if (v_max < 0.0 || !(dt_prev >= 0.0) || !std::isfinite(dt_prev) || !std::isfinite(remaining)) return SPHK_ERR_INVALID;
    int flags = 0;
    double dt;
    if (!std::isfinite(v_max)) {                  // NaN or +inf
        dt = r->dt_min;
        flags |= SPHK_DT_NONFINITE;
    } else {
        const double vb = v_max + r->gravity * dt_prev;
        dt = vb > 0.0 ? r->cfl * r->radius / vb : r->dt_max;
        if (dt > r->dt_max) dt = r->dt_max;
        if (dt < r->dt_min) { dt = r->dt_min; flags |= SPHK_DT_MIN_CLAMP; }
    }
    if (remaining > 0.0) {
        if (remaining <= dt) { dt = remaining; flags |= SPHK_DT_FRAME_END; }
        else if (remaining < 2.0 * dt) dt = 0.5 * remaining;
    }
    *dt_out = static_cast<float>(dt);
    *flags_out = flags;
    return SPHK_OK;
}

static int speed_alloc(sphk_ctx* c) {
    if (c->speedDev) return SPHK_OK;
    cudaError_t e = dalloc(&c->speedDev, 3);
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&c->speedPinned), 3 * sizeof(unsigned int));
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&c->speedEvent, cudaEventDisableTiming);
    if (e != cudaSuccess) {
        cudaFree(c->speedDev); c->speedDev = nullptr;
        if (c->speedPinned) cudaFreeHost(c->speedPinned);
        c->speedPinned = nullptr;
        if (c->speedEvent) cudaEventDestroy(c->speedEvent);
        c->speedEvent = nullptr;
        cudaGetLastError();
        return e == cudaErrorMemoryAllocation ? SPHK_ERR_ALLOC : static_cast<int>(e);
    }
    return SPHK_OK;
}

extern "C" int sphk_step_speed(sphk_ctx* c, const sphk_particles* fluid, int with_bodies) {
    if (!c || !fluid || !fluid->vel || fluid->n < 0 || fluid->n > c->capF) return SPHK_ERR_INVALID;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;
    if (with_bodies && !c->bodies) return SPHK_ERR_STATE;
    const int rc = speed_alloc(c);
    if (rc != SPHK_OK) return rc;
    const int nBodies = with_bodies ? c->bodies->nBodies : 0;
    BodyRadii R{};
    for (int b = 0; b < nBodies; ++b) R.r[b] = c->bodies->rmax[b];
    SPHK_CUDA_TRY(cudaMemsetAsync(c->speedDev, 0, 3 * sizeof(unsigned int), c->stream));
    if (fluid->n > 0 || nBodies > 0) {
        const int blocks = std::max(1, std::min(sphk_blocks(fluid->n), 8 * std::max(c->numSMs, 1)));
        k_step_speed<<<blocks, SPHK_BLOCK, 0, c->stream>>>(fluid->vel, fluid->n, nBodies ? c->bodies->motion : nullptr, nBodies, R,
                                                           c->speedDev);
        c->launches++;
    }
    SPHK_CUDA_TRY(cudaMemcpyAsync(c->speedPinned, c->speedDev, 3 * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaEventRecord(c->speedEvent, c->stream));
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_step_speed_result(sphk_ctx* c, float* v_max_host, int* nonfinite_host) {
    if (!c || !v_max_host || !nonfinite_host) return SPHK_ERR_INVALID;
    if (!c->speedEvent) return SPHK_ERR_STATE;
    SPHK_CUDA_TRY(cudaEventSynchronize(c->speedEvent));
    float v2, b;
    std::memcpy(&v2, c->speedPinned, sizeof(float));
    std::memcpy(&b, c->speedPinned + 1, sizeof(float));
    v_max_host[0] = std::sqrt(v2);
    v_max_host[1] = b;
    *nonfinite_host = static_cast<int>(c->speedPinned[2]);
    return SPHK_OK;
}
