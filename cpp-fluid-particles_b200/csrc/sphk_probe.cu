// sphk_probe.cu -- probes and water-level gauges: SPH-interpolated fluid fields at points, on lattices and along segments, and a
// device-side ring that records them every step (DESIGN.md section 2.13).
//
// Every query reads the API arrays as the step left them (pos, vel, mass, density, the optional pressure and temperature) and the
// fluid cell ranges of the last search, never the packed records.  One thread walks the cell rows around its point in the sweeps'
// row order (dx outermost, then dy, then the contiguous z range), so a point's sums are formed in a fixed order: every layer and
// every execution path gets the same bits for the same state.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <climits>
#include <algorithm>
#include <vector>
#include <math_constants.h>
#include "sphk_internal.cuh"

namespace sphk_probe_detail {

struct ProbeScene {
    const float* __restrict__ pos;
    const float* __restrict__ vel;
    const float* __restrict__ mass;
    const float* __restrict__ density;
    const float* __restrict__ pressure;      // nullptr: p = NaN
    const float* __restrict__ temperature;   // nullptr: T = NaN
    const int* __restrict__ csF;
    int3 cs, org;
    float cellLength;
    float R2;         // R^2: a particle counts when |x - x_j|^2 <= R^2
    float hInv, cW;   // the cubic spline of radius R (as w_cubic, without its r < eps h cut)
    int reach;        // cell rows walked around the point's cell: 2 when positions moved since the search, else 1
};

struct GaugeSet {
    sphk_gauge g[SPHK_GAUGE_LIMIT];
    int n;
    float threshold;
};

// the continuous cubic spline: w_cubic without quirk Q1 (W(0) = cW * 4, so a probe on a particle sees it)
__device__ __forceinline__ float w_probe(float r, const ProbeScene& s) {
    const float q = r * s.hInv;
    const float t = 2.0f - q;
    const float w = (q > 1.0f) ? t * t * t : ((3.0f * q - 6.0f) * q * q + 4.0f);
    return (q > 2.0f) ? 0.0f : s.cW * w;
}

// The sums of one point.  kFull = false: the Shepard sum S only (gauges).  Dry (no particle within R, or the point outside the
// grid): n = 0.  Particles without a positive density have no volume and are skipped.
template <bool kFull>
__device__ __forceinline__ void probe_sums(const ProbeScene& s, float3 x, float& S, float& M, float3& V, float& P, float& T, int& n) {
    S = 0.f; M = 0.f; V = make_float3(0.f, 0.f, 0.f); P = 0.f; T = 0.f; n = 0;
    if (!(x.x - x.x == 0.f && x.y - x.y == 0.f && x.z - x.z == 0.f)) return;
    const int cx = cell_coord(x.x, s.cellLength) - s.org.x, cy = cell_coord(x.y, s.cellLength) - s.org.y,
              cz = cell_coord(x.z, s.cellLength) - s.org.z;
    if (cx < 0 || cx >= s.cs.x || cy < 0 || cy >= s.cs.y || cz < 0 || cz >= s.cs.z) return;
    const int zlo = max(cz - s.reach, 0), zhi = min(cz + s.reach, s.cs.z - 1);
#pragma unroll 1
    for (int ix = max(cx - s.reach, 0); ix <= min(cx + s.reach, s.cs.x - 1); ++ix)
#pragma unroll 1
        for (int iy = max(cy - s.reach, 0); iy <= min(cy + s.reach, s.cs.y - 1); ++iy) {
            const int c0 = (ix * s.cs.y + iy) * s.cs.z;
            const int end = s.csF[c0 + zhi + 1];
            for (int j = s.csF[c0 + zlo]; j < end; ++j) {
                const float3 d = x - load3(s.pos, j);
                const float r2 = dot3(d, d);
                if (!(r2 <= s.R2)) continue;
                const float rho = s.density[j];
                if (!(rho > 0.f)) continue;
                ++n;
                const float m = s.mass[j];
                const float w = w_probe(sqrtf(r2), s);
                const float vw = (m / rho) * w;
                S += vw;
                if (kFull) {
                    M += m * w;
                    V += vw * load3(s.vel, j);
                    if (s.pressure) P += vw * s.pressure[j];
                    if (s.temperature) T += vw * s.temperature[j];
                }
            }
        }
}

// record {S, rho, vx, vy, vz, p, T, n} of point x into out[0..7] (two float4 stores)
__device__ __forceinline__ void probe_record(const ProbeScene& s, float3 x, float* __restrict__ out) {
    float S, M, P, T; float3 V; int n;
    probe_sums<true>(s, x, S, M, V, P, T, n);
    const float inv = S > 0.f ? 1.0f / S : 0.f;
    const float nan = CUDART_NAN_F;
    float4 lo, hi;
    lo.x = S; lo.y = M * inv; lo.z = V.x * inv; lo.w = V.y * inv;
    hi.x = V.z * inv;
    hi.y = s.pressure ? P * inv : nan;
    hi.z = s.temperature ? T * inv : nan;
    hi.w = static_cast<float>(n);
    reinterpret_cast<float4*>(out)[0] = lo;
    reinterpret_cast<float4*>(out)[1] = hi;
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_probe_points(const ProbeScene s, const float* __restrict__ points, int n, float* __restrict__ out) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    probe_record(s, load3(points, i), out + 8 * static_cast<size_t>(i));
}

// lattice point t (z fastest): origin + spacing * (ix, iy, iz), multiply then add, rounded per operation (no contraction)
__global__ void __launch_bounds__(SPHK_BLOCK)
k_probe_lattice(const ProbeScene s, float3 origin, float spacing, int ny, int nz, long long total, float* __restrict__ out) {
    const long long t = static_cast<long long>(blockIdx.x) * SPHK_BLOCK + threadIdx.x;
    if (t >= total) return;
    const int iz = static_cast<int>(t % nz);
    const long long r = t / nz;
    const int iy = static_cast<int>(r % ny);
    const int ix = static_cast<int>(r / ny);
    const float3 x = f3(__fadd_rn(origin.x, __fmul_rn(spacing, static_cast<float>(ix))),
                        __fadd_rn(origin.y, __fmul_rn(spacing, static_cast<float>(iy))),
                        __fadd_rn(origin.z, __fmul_rn(spacing, static_cast<float>(iz))));
    probe_record(s, x, out + 8 * static_cast<size_t>(t));
}

// sample i of gauge g: a + (b - a) * (i / (k - 1)), each operation rounded once
__device__ __forceinline__ float3 gauge_point(const sphk_gauge& g, int i) {
    const float t = __fdiv_rn(static_cast<float>(i), static_cast<float>(g.samples - 1));
    return f3(__fadd_rn(g.a[0], __fmul_rn(__fsub_rn(g.b[0], g.a[0]), t)),
              __fadd_rn(g.a[1], __fmul_rn(__fsub_rn(g.b[1], g.a[1]), t)),
              __fadd_rn(g.a[2], __fmul_rn(__fsub_rn(g.b[2], g.a[2]), t)));
}

__device__ __forceinline__ float gauge_S(const ProbeScene& s, const sphk_gauge& g, int i) {
    float S, M, P, T; float3 V; int n;
    probe_sums<false>(s, gauge_point(g, i), S, M, V, P, T, n);
    return S;
}

// One block per gauge: the block's threads form S at every sample into shared memory (all walks in flight at once), then its first
// warp scans the samples in chunks of 32 from the top down: the first chunk with a wet sample (S >= theta) holds i*, the highest one
// (its ballot's top bit).  Level: the linear crossing of theta between i* and i* + 1 times |b - a| / (k - 1); |b - a| when
// i* = k - 1; -1 when dry.  Called by every thread of the block.
__device__ __forceinline__ void gauge_level(const ProbeScene& s, const sphk_gauge& g, float theta, float* __restrict__ out) {
    __shared__ float sh[SPHK_GAUGE_MAX_SAMPLES];
    const int k = g.samples;
    for (int i = threadIdx.x; i < k; i += blockDim.x) sh[i] = gauge_S(s, g, i);
    __syncthreads();
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    float level = -1.0f;
    for (int c = (k - 1) >> 5; c >= 0; --c) {
        const int i = (c << 5) + lane;
        const unsigned int wet = __ballot_sync(0xffffffffu, i < k && sh[i] >= theta);
        if (wet) {
            const int is = (c << 5) + 31 - __clz(wet);
            const float dx = __fsub_rn(g.b[0], g.a[0]), dy = __fsub_rn(g.b[1], g.a[1]), dz = __fsub_rn(g.b[2], g.a[2]);
            const float L = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            if (is == k - 1) level = L;
            else {
                const float si = sh[is], sn = sh[is + 1];
                const float f = __fdiv_rn(__fsub_rn(si, theta), __fsub_rn(si, sn));
                level = __fdiv_rn(__fmul_rn(L, __fadd_rn(static_cast<float>(is), f)), static_cast<float>(k - 1));
            }
            break;
        }
    }
    if (lane == 0) *out = level;
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_gauge_levels(const ProbeScene s, const GaugeSet gs, float* __restrict__ out) {
    gauge_level(s, gs.g[blockIdx.x], gs.threshold, out + blockIdx.x);
}

// One row of a series: the probe records into slot (*counter mod capacity), then the gauge levels (one block per gauge after the
// probes' blocks), all read from the device counter.  k_series_bump advances it afterwards.
__global__ void __launch_bounds__(SPHK_BLOCK)
k_series_record(const ProbeScene s, const float* __restrict__ points, int nP, int probeBlocks, const GaugeSet gs, int capacity,
                const long long* __restrict__ counter, float* __restrict__ records, float* __restrict__ levels) {
    const long long slot = *counter % capacity;
    if (static_cast<int>(blockIdx.x) < probeBlocks) {
        const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
        if (i < nP) probe_record(s, load3(points, i), records + (slot * nP + i) * 8);
    } else {
        const int w = blockIdx.x - probeBlocks;
        gauge_level(s, gs.g[w], gs.threshold, levels + slot * gs.n + w);
    }
}
__global__ void k_series_bump(long long* counter) { ++*counter; }

__global__ void k_points_finite(const float* __restrict__ p, long long n3, int* __restrict__ bad) {
    for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n3; i += static_cast<long long>(gridDim.x) * blockDim.x)
        if (!(p[i] - p[i] == 0.f)) *bad = 1;
}

static bool finite(float x) { return x - x == 0.f; }

// [a, a + na) and [b, b + nb) (bytes) overlap
static bool overlaps(const void* a, size_t na, const void* b, size_t nb) {
    if (!a || !b || na == 0 || nb == 0) return false;
    const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return x < y + nb && y < x + na;
}

// an output of out_bytes that overlaps a scene array or an input of the call
static bool aliases_scene(const void* out, size_t bytes, const sphk_scene* s, const float* pressure, const float* temperature) {
    const size_t nF = static_cast<size_t>(s->fluid.n), nB = static_cast<size_t>(s->boundary.n);
    return overlaps(out, bytes, s->fluid.pos, 12 * nF) || overlaps(out, bytes, s->fluid.vel, 12 * nF) ||
           overlaps(out, bytes, s->fluid.mass, 4 * nF) || overlaps(out, bytes, s->fluid.density, 4 * nF) ||
           overlaps(out, bytes, s->fluid.pressure, 4 * nF) || overlaps(out, bytes, s->fluid.particle2cell, 4 * nF) ||
           overlaps(out, bytes, s->boundary.pos, 12 * nB) || overlaps(out, bytes, s->boundary.vel, 12 * nB) ||
           overlaps(out, bytes, s->boundary.mass, 4 * nB) || overlaps(out, bytes, s->boundary.density, 4 * nB) ||
           overlaps(out, bytes, s->boundary.pressure, 4 * nB) || overlaps(out, bytes, pressure, 4 * nF) ||
           overlaps(out, bytes, temperature, 4 * nF) || overlaps(out, bytes, s->cell_start_fluid, 4) ||
           overlaps(out, bytes, s->cell_start_boundary, 4);
}

// the scene checks every probe entry shares: searched sets of the scene's sizes, the arrays a probe reads, no slab rank
static int check_probe_scene(const sphk_ctx* c, const sphk_scene* s) {
    if (!c || !s) return SPHK_ERR_INVALID;
    if (!s->cell_start_fluid || !s->fluid.pos || !s->fluid.vel || !s->fluid.mass || !s->fluid.density) return SPHK_ERR_INVALID;
    if (!(s->radius > 0.f) || !finite(s->radius)) return SPHK_ERR_INVALID;
    if (c->actCount >= 0 || c->rangeDev) return SPHK_ERR_STATE;      // slab ranks: a probe near a cut would miss the other rank's fluid
    if (!c->fluidSearched || s->fluid.n != c->nF) return SPHK_ERR_STATE;
    return SPHK_OK;
}

static ProbeScene probe_scene(const sphk_ctx* c, const sphk_scene* s, const float* pressure, const float* temperature) {
    ProbeScene p;
    p.pos = s->fluid.pos; p.vel = s->fluid.vel; p.mass = s->fluid.mass; p.density = s->fluid.density;
    p.pressure = pressure; p.temperature = temperature;
    p.csF = s->cell_start_fluid;
    p.cs = c->cs; p.org = c->org; p.cellLength = c->cellLength;
    const float R = s->radius;
    p.R2 = R * R;
    p.hInv = static_cast<float>(2.0 / R);
    p.cW = static_cast<float>(0.25 / (3.14159265358979323846 * R * R * R));
    // the cell ranges are those of the search: a particle moved since (PBD corrections, advection) by up to one cell may be
    // listed one row further out
    p.reach = c->posDirty ? 2 : 1;
    return p;
}

static int check_gauges(const sphk_gauge* g, int n, float threshold) {
    if (!g || n < 1 || n > SPHK_GAUGE_LIMIT || !finite(threshold) || !(threshold > 0.f)) return SPHK_ERR_INVALID;
    for (int i = 0; i < n; ++i) {
        bool same = true;
        for (int a = 0; a < 3; ++a) {
            if (!finite(g[i].a[a]) || !finite(g[i].b[a])) return SPHK_ERR_INVALID;
            same = same && g[i].a[a] == g[i].b[a];
        }
        if (same || g[i].samples < 2 || g[i].samples > SPHK_GAUGE_MAX_SAMPLES) return SPHK_ERR_INVALID;
    }
    return SPHK_OK;
}

static GaugeSet gauge_set(const sphk_gauge* g, int n, float threshold) {
    GaugeSet gs;
    std::memset(&gs, 0, sizeof(gs));
    for (int i = 0; i < n; ++i) gs.g[i] = g[i];
    gs.n = n;
    gs.threshold = threshold;
    return gs;
}

}  // namespace sphk_probe_detail
using namespace sphk_probe_detail;

struct sphk_probe_series {
    cudaStream_t stream = nullptr;
    int nP = 0, capacity = 0;
    float* points = nullptr;       // device float3[nP]
    GaugeSet gauges{};
    float* records = nullptr;      // device [capacity][nP][8]
    float* levels = nullptr;       // device [capacity][nG]
    long long* counter = nullptr;  // device: rows recorded so far
};

extern "C" int sphk_probe_sample(sphk_ctx* c, const sphk_scene* s, const float* points, int n, const float* pressure_or_null,
                                 const float* temperature_or_null, float* out) {
    const int rc = check_probe_scene(c, s);
    if (rc != SPHK_OK) return rc;
    if (n < 0 || (n > 0 && (!points || !out))) return SPHK_ERR_INVALID;
    if (n == 0) return SPHK_OK;
    const size_t bytes = 32 * static_cast<size_t>(n);
    if (aliases_scene(out, bytes, s, pressure_or_null, temperature_or_null) || overlaps(out, bytes, points, 12 * static_cast<size_t>(n)))
        return SPHK_ERR_INVALID;
    if (reinterpret_cast<uintptr_t>(out) % 16) return SPHK_ERR_INVALID;     // two float4 stores per record
    // the points live on the device: a finite check there, read back before anything is written
    int* bad = reinterpret_cast<int*>(c->partial);
    SPHK_CUDA_TRY(cudaMemsetAsync(bad, 0, sizeof(int), c->stream));
    k_points_finite<<<static_cast<int>(std::min<long long>(1024, (3LL * n + SPHK_BLOCK - 1) / SPHK_BLOCK)), SPHK_BLOCK, 0, c->stream>>>(points, 3LL * n, bad);
    int hbad = 0;
    SPHK_CUDA_TRY(cudaMemcpyAsync(&hbad, bad, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->launches++;
    if (hbad) return SPHK_ERR_INVALID;
    k_probe_points<<<sphk_blocks(n), SPHK_BLOCK, 0, c->stream>>>(probe_scene(c, s, pressure_or_null, temperature_or_null), points, n, out);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_probe_lattice(sphk_ctx* c, const sphk_scene* s, const float origin[3], float spacing, const int dims[3],
                                  const float* pressure_or_null, const float* temperature_or_null, float* out) {
    const int rc = check_probe_scene(c, s);
    if (rc != SPHK_OK) return rc;
    if (!origin || !dims || !out || !finite(spacing) || !(spacing > 0.f)) return SPHK_ERR_INVALID;
    long long total = 1;
    for (int a = 0; a < 3; ++a) {
        if (!finite(origin[a]) || dims[a] < 1) return SPHK_ERR_INVALID;
        total *= dims[a];
        if (total > INT_MAX) return SPHK_ERR_INVALID;
    }
    const size_t bytes = 32 * static_cast<size_t>(total);
    if (aliases_scene(out, bytes, s, pressure_or_null, temperature_or_null) || reinterpret_cast<uintptr_t>(out) % 16) return SPHK_ERR_INVALID;
    const long long blocks = (total + SPHK_BLOCK - 1) / SPHK_BLOCK;
    k_probe_lattice<<<static_cast<unsigned int>(blocks), SPHK_BLOCK, 0, c->stream>>>(
        probe_scene(c, s, pressure_or_null, temperature_or_null), make_float3(origin[0], origin[1], origin[2]), spacing, dims[1], dims[2], total, out);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_gauge_levels(sphk_ctx* c, const sphk_scene* s, const sphk_gauge* gauges, int n_gauges, float threshold, float* out) {
    const int rc = check_probe_scene(c, s);
    if (rc != SPHK_OK) return rc;
    if (!out || check_gauges(gauges, n_gauges, threshold) != SPHK_OK) return SPHK_ERR_INVALID;
    if (aliases_scene(out, 4 * static_cast<size_t>(n_gauges), s, nullptr, nullptr)) return SPHK_ERR_INVALID;
    k_gauge_levels<<<n_gauges, SPHK_BLOCK, 0, c->stream>>>(probe_scene(c, s, nullptr, nullptr),
                                                                                              gauge_set(gauges, n_gauges, threshold), out);
    c->launches++;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_probe_series_create(sphk_probe_series** out, const float* points_host, int n_points, const sphk_gauge* gauges_host,
                                        int n_gauges, float threshold, int capacity, void* stream) {
    if (!out) return SPHK_ERR_INVALID;
    *out = nullptr;
    if (n_points < 0 || n_points > SPHK_PROBE_LIMIT || (n_points > 0 && !points_host) || n_gauges < 0 || n_gauges > SPHK_GAUGE_LIMIT ||
        (n_points == 0 && n_gauges == 0) || capacity < 1 || capacity > SPHK_PROBE_CAPACITY_LIMIT)
        return SPHK_ERR_INVALID;
    for (long long i = 0; i < 3LL * n_points; ++i)
        if (!finite(points_host[i])) return SPHK_ERR_INVALID;
    if (n_gauges > 0 && check_gauges(gauges_host, n_gauges, threshold) != SPHK_OK) return SPHK_ERR_INVALID;
    if (n_gauges == 0 && !(finite(threshold) && threshold > 0.f)) return SPHK_ERR_INVALID;
    int dev = 0;
    if (cudaGetDeviceCount(&dev) != cudaSuccess || dev < 1) { cudaGetLastError(); return SPHK_ERR_NO_DEVICE; }
    auto* q = new sphk_probe_series;
    q->stream = static_cast<cudaStream_t>(stream);
    q->nP = n_points; q->capacity = capacity;
    q->gauges = gauge_set(gauges_host, n_gauges, threshold);
    bool ok = cudaMalloc(&q->counter, sizeof(long long)) == cudaSuccess;
    if (ok && n_points > 0) ok = cudaMalloc(&q->points, 12 * static_cast<size_t>(n_points)) == cudaSuccess &&
                                 cudaMalloc(&q->records, 32 * static_cast<size_t>(n_points) * capacity) == cudaSuccess;
    if (ok && n_gauges > 0) ok = cudaMalloc(&q->levels, 4 * static_cast<size_t>(n_gauges) * capacity) == cudaSuccess;
    if (ok && n_points > 0) ok = cudaMemcpy(q->points, points_host, 12 * static_cast<size_t>(n_points), cudaMemcpyHostToDevice) == cudaSuccess;
    if (ok) ok = cudaMemset(q->counter, 0, sizeof(long long)) == cudaSuccess;
    if (!ok) { cudaGetLastError(); sphk_probe_series_destroy(q); return SPHK_ERR_ALLOC; }
    *out = q;
    return SPHK_OK;
}

extern "C" void sphk_probe_series_destroy(sphk_probe_series* q) {
    if (!q) return;
    if (q->stream) cudaStreamSynchronize(q->stream);
    cudaFree(q->points); cudaFree(q->records); cudaFree(q->levels); cudaFree(q->counter);
    delete q;
}

extern "C" int sphk_probes_record(sphk_ctx* c, const sphk_scene* s, sphk_probe_series* q, const float* pressure_or_null,
                                  const float* temperature_or_null) {
    const int rc = check_probe_scene(c, s);
    if (rc != SPHK_OK) return rc;
    if (!q) return SPHK_ERR_INVALID;
    const int probeBlocks = sphk_blocks(q->nP);
    const int gaugeBlocks = q->gauges.n;
    k_series_record<<<probeBlocks + gaugeBlocks, SPHK_BLOCK, 0, c->stream>>>(probe_scene(c, s, pressure_or_null, temperature_or_null),
                                                                             q->points, q->nP, probeBlocks, q->gauges, q->capacity,
                                                                             q->counter, q->records, q->levels);
    k_series_bump<<<1, 1, 0, c->stream>>>(q->counter);
    c->launches += 2;
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_probe_series_read(sphk_probe_series* q, long long* count, int max_rows, float* records_host, float* levels_host,
                                      int* rows_out) {
    if (!q || !count || !rows_out || max_rows < 0) return SPHK_ERR_INVALID;
    SPHK_CUDA_TRY(cudaMemcpyAsync(count, q->counter, sizeof(long long), cudaMemcpyDeviceToHost, q->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(q->stream));
    const long long avail = std::min<long long>(*count, q->capacity);
    const int rows = static_cast<int>(std::min<long long>(avail, max_rows));
    if (rows > 0 && ((q->nP > 0 && !records_host) || (q->gauges.n > 0 && !levels_host))) return SPHK_ERR_INVALID;
    const size_t rec = 8 * static_cast<size_t>(q->nP), lev = static_cast<size_t>(q->gauges.n);
    // the last `rows` rows, oldest first: at most two contiguous runs of slots
    long long slot = (*count - rows) % q->capacity;
    for (int r = 0; r < rows;) {
        const int run = static_cast<int>(std::min<long long>(rows - r, q->capacity - slot));
        if (rec) SPHK_CUDA_TRY(cudaMemcpyAsync(records_host + r * rec, q->records + slot * rec, 4 * rec * run, cudaMemcpyDeviceToHost, q->stream));
        if (lev) SPHK_CUDA_TRY(cudaMemcpyAsync(levels_host + r * lev, q->levels + slot * lev, 4 * lev * run, cudaMemcpyDeviceToHost, q->stream));
        r += run;
        slot = 0;
    }
    SPHK_CUDA_TRY(cudaStreamSynchronize(q->stream));
    *rows_out = rows;
    return SPHK_OK;
}
