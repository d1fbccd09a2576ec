// sphk_mesh.cu -- scenes from triangle meshes (DESIGN.md section 2.12): mass properties on the host in double; on the device
// triangle bins, inside / near classification, lattice fill and Poisson-disk surface sampling.
//
//   bins      : per triangle the cells its bounding box overlaps -> (cell, triangle) pairs in triangle order -> one stable radix
//               sort by cell -> cell ranges.  Two bins: a 3D grid for distances, an (x, z) column grid for the +y ray.
//   classify  : parity of the crossings of the +y ray.  The (x, z) orientation of the point against every edge is evaluated
//               exactly (the six float products of the expanded determinant are exact in double; their sum's sign comes from a
//               nonoverlapping expansion) and a zero is resolved by moving the point by (eps, eps^2): the same perturbation for
//               every triangle, so a ray through a shared edge or vertex is counted as the perturbed ray is, once.
//   fill      : count, scan, write over the lattice of the mesh's bounding box, points formed as sphk_scene_fluid_block forms them.
//   sample    : candidates on a barycentric lattice per triangle, sorted into cells of side r (1 + 1e-5), accepted per cell in
//               candidate order in 27 colour phases (cell index mod 3 per axis: cells of one colour share no neighbour).
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <vector>
#include "sphk_internal.cuh"

struct sphk_mesh {
    int nv = 0, nt = 0, closed = 0;
    float* v = nullptr;                    // float3[nv]
    int* tri = nullptr;                    // int3[nt]
    float lo[3], hi[3];                    // bounding box
    float h3 = 1.f, inv3 = 1.f;            // 3D grid: cell side, its reciprocal, dims
    int d3[3] = {1, 1, 1};
    int* start3 = nullptr;                 // int[cells + 1]
    int* items3 = nullptr;                 // triangle indices, grouped by cell, ascending within a cell
    float h2 = 1.f, inv2 = 1.f;            // column grid over (x, z)
    int d2[2] = {1, 1};
    int* start2 = nullptr;
    int* items2 = nullptr;
    cudaStream_t stream = nullptr;
};

namespace {

struct MeshDev {
    const float* v;
    const int* tri;
    float ox, oy, oz;
    float inv3; int dx, dy, dz; const int* start3; const int* items3;
    float inv2; int cx, cz; const int* start2; const int* items2;
};

MeshDev dev_of(const sphk_mesh* m) {
    return MeshDev{m->v, m->tri, m->lo[0], m->lo[1], m->lo[2], m->inv3, m->d3[0], m->d3[1], m->d3[2], m->start3, m->items3,
                   m->inv2, m->d2[0], m->d2[1], m->start2, m->items2};
}

// the cell of coordinate x: monotone in x (subtract, multiply, floor, clamp), the same function for binning and lookup
__host__ __device__ __forceinline__ int cell_of(float x, float o, float inv, int d) {
    float f = floorf((x - o) * inv);
    f = fminf(fmaxf(f, 0.f), static_cast<float>(d - 1));
    return static_cast<int>(f);
}

__device__ __forceinline__ float3 vtx(const float* v, int i) { return make_float3(v[3 * i], v[3 * i + 1], v[3 * i + 2]); }
__device__ __forceinline__ float dot(float3 a, float3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ float length(float3 a) { return sqrtf(dot(a, a)); }

// ---- bins --------------------------------------------------------------------------------------------------------------------
// mode 3: cells of the 3D grid; mode 2: columns of the (x, z) grid
template <int MODE>
__device__ __forceinline__ void tri_cells(const MeshDev& m, int t, int3& a, int3& b) {
    const int i0 = m.tri[3 * t], i1 = m.tri[3 * t + 1], i2 = m.tri[3 * t + 2];
    const float3 p = vtx(m.v, i0), q = vtx(m.v, i1), r = vtx(m.v, i2);
    const float lx = fminf(p.x, fminf(q.x, r.x)), hx = fmaxf(p.x, fmaxf(q.x, r.x));
    const float ly = fminf(p.y, fminf(q.y, r.y)), hy = fmaxf(p.y, fmaxf(q.y, r.y));
    const float lz = fminf(p.z, fminf(q.z, r.z)), hz = fmaxf(p.z, fmaxf(q.z, r.z));
    if (MODE == 3) {
        a = make_int3(cell_of(lx, m.ox, m.inv3, m.dx), cell_of(ly, m.oy, m.inv3, m.dy), cell_of(lz, m.oz, m.inv3, m.dz));
        b = make_int3(cell_of(hx, m.ox, m.inv3, m.dx), cell_of(hy, m.oy, m.inv3, m.dy), cell_of(hz, m.oz, m.inv3, m.dz));
    } else {
        a = make_int3(cell_of(lx, m.ox, m.inv2, m.cx), 0, cell_of(lz, m.oz, m.inv2, m.cz));
        b = make_int3(cell_of(hx, m.ox, m.inv2, m.cx), 0, cell_of(hz, m.oz, m.inv2, m.cz));
    }
}

template <int MODE>
__global__ void __launch_bounds__(SPHK_BLOCK) k_bin_count(MeshDev m, int nt, long long* counts) {
    const int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (t >= nt) return;
    int3 a, b;
    tri_cells<MODE>(m, t, a, b);
    counts[t] = static_cast<long long>(b.x - a.x + 1) * (b.y - a.y + 1) * (b.z - a.z + 1);
}

template <int MODE>
__global__ void __launch_bounds__(SPHK_BLOCK) k_bin_write(MeshDev m, int nt, const long long* offsets, int* keys, int* vals) {
    const int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (t >= nt) return;
    int3 a, b;
    tri_cells<MODE>(m, t, a, b);
    long long o = offsets[t];
    for (int x = a.x; x <= b.x; ++x)
        for (int y = a.y; y <= b.y; ++y)
            for (int z = a.z; z <= b.z; ++z) {
                keys[o] = MODE == 3 ? (x * m.dy + y) * m.dz + z : x * m.cz + z;
                vals[o] = t;
                ++o;
            }
}

// start[c] = first sorted pair with key >= c, c in [0, cells]
__global__ void __launch_bounds__(SPHK_BLOCK) k_bin_start(const int* keys, int n, int cells, int* start) {
    const int c = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (c > cells) return;
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (keys[mid] < c) lo = mid + 1; else hi = mid;
    }
    start[c] = lo;
}

// ---- exact (x, z) orientation --------------------------------------------------------------------------------------------------
__device__ __forceinline__ void two_sum(double a, double b, double& s, double& e) {
    s = __dadd_rn(a, b);
    const double bb = __dsub_rn(s, a);
    e = __dadd_rn(__dsub_rn(a, __dsub_rn(s, bb)), __dsub_rn(b, bb));
}

// sign of sum x[0..5] exactly (Shewchuk's grow-expansion: nonoverlapping components of increasing magnitude; the sign is that of
// the largest nonzero one)
__device__ int exact_sign6(const double* x) {
    double h[6];
    int n = 0;
    for (int k = 0; k < 6; ++k) {
        double q = x[k];
        for (int i = 0; i < n; ++i) {
            double s, e;
            two_sum(q, h[i], s, e);
            h[i] = e;
            q = s;
        }
        h[n++] = q;
    }
    for (int i = n - 1; i >= 0; --i)
        if (h[i] != 0.0) return h[i] > 0.0 ? 1 : -1;
    return 0;
}

// sign of (b - a) x (q - a) in the (x, z) plane for the point q moved by (eps, eps^2) -- never 0 unless a == b
__device__ int orient_xz(float ax, float az, float bx, float bz, float qx, float qz) {
    const double t1 = (static_cast<double>(bx) - ax) * (static_cast<double>(qz) - az);
    const double t2 = (static_cast<double>(bz) - az) * (static_cast<double>(qx) - ax);
    const double d = t1 - t2;
    int s;
    if (fabs(d) > 1e-14 * (fabs(t1) + fabs(t2))) {
        s = d > 0.0 ? 1 : -1;
    } else {      // bx qz - bx az - ax qz - bz qx + bz ax + az qx, every product of two floats exact in double
        const double x[6] = {static_cast<double>(bx) * qz, -static_cast<double>(bx) * az, -static_cast<double>(ax) * qz,
                             -static_cast<double>(bz) * qx, static_cast<double>(bz) * ax, static_cast<double>(az) * qx};
        s = exact_sign6(x);
    }
    if (s != 0) return s;
    if (bz != az) return bz < az ? 1 : -1;       // d/dqx = -(bz - az)
    if (bx != ax) return bx > ax ? 1 : -1;       // d/dqz = (bx - ax)
    return 0;
}

__device__ int ray_parity(const MeshDev& m, float3 p) {
    const int col = cell_of(p.x, m.ox, m.inv2, m.cx) * m.cz + cell_of(p.z, m.oz, m.inv2, m.cz);
    int parity = 0;
    for (int s = m.start2[col], e = m.start2[col + 1]; s < e; ++s) {
        const int t = m.items2[s];
        const float3 a = vtx(m.v, m.tri[3 * t]), b = vtx(m.v, m.tri[3 * t + 1]), c = vtx(m.v, m.tri[3 * t + 2]);
        const int s0 = orient_xz(a.x, a.z, b.x, b.z, p.x, p.z);
        if (s0 == 0) continue;
        if (orient_xz(b.x, b.z, c.x, c.z, p.x, p.z) != s0 || orient_xz(c.x, c.z, a.x, a.z, p.x, p.z) != s0) continue;
        // the crossing is above p when n . (a - p) and the projected orientation s0 have opposite signs (n = (b - a) x (c - a),
        // n.y = -s0 |n.y|); p on the triangle itself is within any clearance, so this test needs no exact arithmetic
        const double ux = static_cast<double>(b.x) - a.x, uy = static_cast<double>(b.y) - a.y, uz = static_cast<double>(b.z) - a.z;
        const double vx = static_cast<double>(c.x) - a.x, vy = static_cast<double>(c.y) - a.y, vz = static_cast<double>(c.z) - a.z;
        const double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
        const double f = nx * (static_cast<double>(a.x) - p.x) + ny * (static_cast<double>(a.y) - p.y) + nz * (static_cast<double>(a.z) - p.z);
        if (s0 * f < 0.0) parity ^= 1;
    }
    return parity;
}

// squared distance from p to triangle abc (closest point by Voronoi region, Ericson 5.1.5)
__device__ float dist2_tri(float3 p, float3 a, float3 b, float3 c) {
    const float3 ab = b - a, ac = c - a, ap = p - a;
    const float d1 = dot(ab, ap), d2 = dot(ac, ap);
    float3 q;
    if (d1 <= 0.f && d2 <= 0.f) { q = a; }
    else {
        const float3 bp = p - b;
        const float d3 = dot(ab, bp), d4 = dot(ac, bp);
        if (d3 >= 0.f && d4 <= d3) { q = b; }
        else {
            const float vc = d1 * d4 - d3 * d2;
            if (vc <= 0.f && d1 >= 0.f && d3 <= 0.f) { q = a + (d1 / (d1 - d3)) * ab; }
            else {
                const float3 cp = p - c;
                const float d5 = dot(ab, cp), d6 = dot(ac, cp);
                if (d6 >= 0.f && d5 <= d6) { q = c; }
                else {
                    const float vb = d5 * d2 - d1 * d6;
                    if (vb <= 0.f && d2 >= 0.f && d6 <= 0.f) { q = a + (d2 / (d2 - d6)) * ac; }
                    else {
                        const float va = d3 * d6 - d5 * d4;
                        if (va <= 0.f && (d4 - d3) >= 0.f && (d5 - d6) >= 0.f) { q = b + ((d4 - d3) / ((d4 - d3) + (d5 - d6))) * (c - b); }
                        else {
                            const float den = 1.f / (va + vb + vc);
                            q = a + ab * (vb * den) + ac * (vc * den);
                        }
                    }
                }
            }
        }
    }
    const float3 d = p - q;
    return dot(d, d);
}

__device__ bool near_surface(const MeshDev& m, float3 p, float clearance) {
    const float c2 = clearance * clearance;
    const int x0 = cell_of(p.x - clearance, m.ox, m.inv3, m.dx), x1 = cell_of(p.x + clearance, m.ox, m.inv3, m.dx);
    const int y0 = cell_of(p.y - clearance, m.oy, m.inv3, m.dy), y1 = cell_of(p.y + clearance, m.oy, m.inv3, m.dy);
    const int z0 = cell_of(p.z - clearance, m.oz, m.inv3, m.dz), z1 = cell_of(p.z + clearance, m.oz, m.inv3, m.dz);
    for (int x = x0; x <= x1; ++x)
        for (int y = y0; y <= y1; ++y)
            for (int z = z0; z <= z1; ++z) {
                const int cell = (x * m.dy + y) * m.dz + z;
                for (int s = m.start3[cell], e = m.start3[cell + 1]; s < e; ++s) {
                    const int t = m.items3[s];
                    if (dist2_tri(p, vtx(m.v, m.tri[3 * t]), vtx(m.v, m.tri[3 * t + 1]), vtx(m.v, m.tri[3 * t + 2])) <= c2) return true;
                }
            }
    return false;
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_mesh_classify(MeshDev m, const float* pos, int n, float clearance, int* flags) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float3 p = make_float3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
    flags[i] = (ray_parity(m, p) ? SPHK_MESH_INSIDE : 0) | (near_surface(m, p, clearance) ? SPHK_MESH_NEAR : 0);
}

// ---- fill ------------------------------------------------------------------------------------------------------------------------
struct Lattice {
    float ox, oy, oz, s;
    int j0, i0, k0, nx, ny, nz;       // index ranges [j0, j0 + nx) x [i0, i0 + ny) x [k0, k0 + nz)
};

__device__ __forceinline__ float3 lattice_point(const Lattice& L, int idx) {
    const int k = L.k0 + idx % L.nz;
    const int q = idx / L.nz;
    const int j = L.j0 + q % L.nx;
    const int i = L.i0 + q / L.nx;
    return make_float3(__fadd_rn(L.ox, __fmul_rn(L.s, static_cast<float>(j))), __fadd_rn(L.oy, __fmul_rn(L.s, static_cast<float>(i))),
                       __fadd_rn(L.oz, __fmul_rn(L.s, static_cast<float>(k))));
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_fill_flag(MeshDev m, Lattice L, int n, float clearance, int* keep) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    const float3 p = lattice_point(L, i);
    keep[i] = ray_parity(m, p) && !near_surface(m, p, clearance);
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_fill_write(Lattice L, int n, const int* keep, const int* offset, float* out) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n || !keep[i]) return;
    const float3 p = lattice_point(L, i);
    const int o = offset[i];
    out[3 * o] = p.x; out[3 * o + 1] = p.y; out[3 * o + 2] = p.z;
}

// ---- surface sampling ----------------------------------------------------------------------------------------------------------
constexpr int kCellSamples = 16;      // accepted samples per cell: at most 8 points of a cube of side r are r apart

struct SampleGrid {
    float ox, oy, oz, inv;
    long long dx, dy, dz;
};

__device__ __forceinline__ int tri_subdiv(const float* v, const int* tri, int t, float step) {
    const float3 a = vtx(v, tri[3 * t]), b = vtx(v, tri[3 * t + 1]), c = vtx(v, tri[3 * t + 2]);
    const float e = fmaxf(length(b - a), fmaxf(length(c - b), length(a - c)));
    return max(1, static_cast<int>(ceilf(e / step)));
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_cand_count(const float* v, const int* tri, int nt, float step, long long* counts) {
    const int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (t >= nt) return;
    const long long m = tri_subdiv(v, tri, t, step);
    counts[t] = (m + 1) * (m + 2) / 2;
}

__device__ __forceinline__ unsigned long long sample_key(const SampleGrid& g, float3 p) {
    const long long x = static_cast<long long>(fminf(fmaxf(floorf((p.x - g.ox) * g.inv), 0.f), static_cast<float>(g.dx - 1)));
    const long long y = static_cast<long long>(fminf(fmaxf(floorf((p.y - g.oy) * g.inv), 0.f), static_cast<float>(g.dy - 1)));
    const long long z = static_cast<long long>(fminf(fmaxf(floorf((p.z - g.oz) * g.inv), 0.f), static_cast<float>(g.dz - 1)));
    return static_cast<unsigned long long>((x * g.dy + y) * g.dz + z);
}

// candidate (i, j) of triangle t: ((m - i - j) a + i b + j c) / m, i + j <= m, in (i, j) order
__global__ void __launch_bounds__(SPHK_BLOCK)
k_cand_write(const float* v, const int* tri, int nt, float step, SampleGrid g, const long long* offsets, float* cand,
             unsigned long long* keys, int* idx) {
    const int t = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (t >= nt) return;
    const int m = tri_subdiv(v, tri, t, step);
    const float3 a = vtx(v, tri[3 * t]), b = vtx(v, tri[3 * t + 1]), c = vtx(v, tri[3 * t + 2]);
    const float inv = 1.f / static_cast<float>(m);
    long long o = offsets[t];
    for (int i = 0; i <= m; ++i)
        for (int j = 0; i + j <= m; ++j) {
            const float wa = static_cast<float>(m - i - j) * inv, wb = static_cast<float>(i) * inv, wc = static_cast<float>(j) * inv;
            const float3 p = i == m ? b : j == m ? c : (i == 0 && j == 0) ? a : wa * a + wb * b + wc * c;
            cand[3 * o] = p.x; cand[3 * o + 1] = p.y; cand[3 * o + 2] = p.z;
            keys[o] = sample_key(g, p);
            idx[o] = static_cast<int>(o);
            ++o;
        }
}

__global__ void __launch_bounds__(SPHK_BLOCK) k_cell_heads(const unsigned long long* keys, int n, int* head) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n) return;
    head[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_cell_list(const unsigned long long* keys, int n, const int* head, const int* cellOf, unsigned long long* cellKey, int* cellStart) {
    const int i = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (i >= n || !head[i]) return;
    cellKey[cellOf[i]] = keys[i];
    cellStart[cellOf[i]] = i;
}

__device__ __forceinline__ int find_cell(const unsigned long long* cellKey, int nCells, unsigned long long key) {
    int lo = 0, hi = nCells;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (cellKey[mid] < key) lo = mid + 1; else hi = mid;
    }
    return (lo < nCells && cellKey[lo] == key) ? lo : -1;
}

// one thread per cell of colour `phase`: its candidates in order, each accepted when no accepted sample of the 27 cells around is
// closer than r (squared distances in double)
__global__ void __launch_bounds__(SPHK_BLOCK)
k_sample_phase(SampleGrid g, int phase, const unsigned long long* cellKey, const int* cellStart, int nCells, const int* idxSorted,
               const float* cand, double rr, float3* acc, int* accCount, int* accepted, int* overflow) {
    const int cell = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (cell >= nCells) return;
    const unsigned long long key = cellKey[cell];
    const long long cz = static_cast<long long>(key % g.dz), cy = static_cast<long long>((key / g.dz) % g.dy),
                    cx = static_cast<long long>(key / g.dz / g.dy);
    if ((cx % 3) * 9 + (cy % 3) * 3 + cz % 3 != phase) return;
    int nb[27];
    int nn = 0;
    for (long long x = cx - 1; x <= cx + 1; ++x)
        for (long long y = cy - 1; y <= cy + 1; ++y)
            for (long long z = cz - 1; z <= cz + 1; ++z) {
                if (x < 0 || y < 0 || z < 0 || x >= g.dx || y >= g.dy || z >= g.dz) continue;
                const int c = x == cx && y == cy && z == cz ? cell
                                                             : find_cell(cellKey, nCells, static_cast<unsigned long long>((x * g.dy + y) * g.dz + z));
                if (c >= 0) nb[nn++] = c;
            }
    int mine = 0;
    for (int s = cellStart[cell], e = cellStart[cell + 1]; s < e; ++s) {
        const int k = idxSorted[s];
        const float3 p = make_float3(cand[3 * k], cand[3 * k + 1], cand[3 * k + 2]);
        bool ok = true;
        for (int q = 0; q < nn && ok; ++q) {
            const int c = nb[q];
            const int cnt = c == cell ? mine : accCount[c];
            for (int a = 0; a < cnt; ++a) {
                const float3 o = acc[c * kCellSamples + a];
                const double dx = static_cast<double>(p.x) - o.x, dy = static_cast<double>(p.y) - o.y, dz = static_cast<double>(p.z) - o.z;
                if (dx * dx + dy * dy + dz * dz < rr) { ok = false; break; }
            }
        }
        if (!ok) continue;
        if (mine == kCellSamples) { atomicExch(overflow, 1); continue; }
        acc[cell * kCellSamples + mine++] = p;
        accepted[s] = 1;
    }
    accCount[cell] = mine;
}

__global__ void __launch_bounds__(SPHK_BLOCK)
k_sample_write(int n, const int* accepted, const int* offset, const int* idxSorted, const float* cand, float* out) {
    const int s = blockIdx.x * SPHK_BLOCK + threadIdx.x;
    if (s >= n || !accepted[s]) return;
    const int k = idxSorted[s], o = offset[s];
    out[3 * o] = cand[3 * k]; out[3 * o + 1] = cand[3 * k + 1]; out[3 * o + 2] = cand[3 * k + 2];
}

// ---- host helpers -----------------------------------------------------------------------------------------------------------------
bool overlap(const void* a, size_t na, const void* b, size_t nb) {
    const auto x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return x < y + nb && y < x + na;
}

int mesh_check(const float* v, int nv, const int* tri, int nt) {
    if (!v || !tri || nv < 3 || nt < 1 || overlap(v, 12ull * nv, tri, 12ull * nt)) return SPHK_ERR_INVALID;
    for (long long i = 0; i < 3LL * nv; ++i)
        if (!std::isfinite(v[i])) return SPHK_ERR_INVALID;
    for (long long i = 0; i < 3LL * nt; ++i)
        if (tri[i] < 0 || tri[i] >= nv) return SPHK_ERR_INVALID;
    return SPHK_OK;
}

// every undirected edge used exactly twice, once in each direction
bool mesh_closed(const int* tri, int nt) {
    if (nt < 4) return false;
    std::vector<std::pair<unsigned long long, int>> e;
    e.reserve(3ull * nt);
    for (int t = 0; t < nt; ++t)
        for (int k = 0; k < 3; ++k) {
            const unsigned a = static_cast<unsigned>(tri[3 * t + k]), b = static_cast<unsigned>(tri[3 * t + (k + 1) % 3]);
            if (a == b) return false;
            e.push_back({(static_cast<unsigned long long>(std::min(a, b)) << 32) | std::max(a, b), a < b ? 1 : -1});
        }
    std::sort(e.begin(), e.end());
    for (size_t i = 0; i < e.size(); i += 2)
        if (i + 1 >= e.size() || e[i].first != e[i + 1].first || e[i].second + e[i + 1].second != 0 ||
            (i + 2 < e.size() && e[i + 2].first == e[i].first))
            return false;
    return true;
}

// cyclic Jacobi on a symmetric 3x3 matrix: A -> diagonal, V = eigenvectors as columns
void jacobi3(double A[3][3], double V[3][3]) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) V[i][j] = i == j ? 1.0 : 0.0;
    for (int sweep = 0; sweep < 50; ++sweep) {
        const double off = A[0][1] * A[0][1] + A[0][2] * A[0][2] + A[1][2] * A[1][2];
        const double diag = A[0][0] * A[0][0] + A[1][1] * A[1][1] + A[2][2] * A[2][2];
        if (off == 0.0 || off <= 1e-36 * diag) break;
        static const int P[3][2] = {{0, 1}, {0, 2}, {1, 2}};
        for (const auto& pq : P) {
            const int p = pq[0], q = pq[1];
            // an off-diagonal at rounding level (an isotropic body) is 0: its rotation would only turn the axes by noise
            if (std::fabs(A[p][q]) <= 1e-13 * (std::fabs(A[p][p]) + std::fabs(A[q][q]))) { A[p][q] = A[q][p] = 0.0; continue; }
            const double theta = (A[q][q] - A[p][p]) / (2.0 * A[p][q]);
            const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
            const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
            for (int k = 0; k < 3; ++k) {           // columns p, q
                const double akp = A[k][p], akq = A[k][q];
                A[k][p] = c * akp - s * akq; A[k][q] = s * akp + c * akq;
            }
            for (int k = 0; k < 3; ++k) {           // rows p, q
                const double apk = A[p][k], aqk = A[q][k];
                A[p][k] = c * apk - s * aqk; A[q][k] = s * apk + c * aqk;
            }
            A[p][q] = A[q][p] = 0.0;
            for (int k = 0; k < 3; ++k) {
                const double vkp = V[k][p], vkq = V[k][q];
                V[k][p] = c * vkp - s * vkq; V[k][q] = s * vkp + c * vkq;
            }
        }
    }
}

void quat_of(const double R[3][3], double q[4]) {   // R: body axes as columns; q = (x, y, z, w)
    const double tr = R[0][0] + R[1][1] + R[2][2];
    double x, y, z, w;
    if (tr > 0.0) {
        const double S = std::sqrt(tr + 1.0) * 2.0;
        w = 0.25 * S; x = (R[2][1] - R[1][2]) / S; y = (R[0][2] - R[2][0]) / S; z = (R[1][0] - R[0][1]) / S;
    } else if (R[0][0] > R[1][1] && R[0][0] > R[2][2]) {
        const double S = std::sqrt(1.0 + R[0][0] - R[1][1] - R[2][2]) * 2.0;
        w = (R[2][1] - R[1][2]) / S; x = 0.25 * S; y = (R[0][1] + R[1][0]) / S; z = (R[0][2] + R[2][0]) / S;
    } else if (R[1][1] > R[2][2]) {
        const double S = std::sqrt(1.0 + R[1][1] - R[0][0] - R[2][2]) * 2.0;
        w = (R[0][2] - R[2][0]) / S; x = (R[0][1] + R[1][0]) / S; y = 0.25 * S; z = (R[1][2] + R[2][1]) / S;
    } else {
        const double S = std::sqrt(1.0 + R[2][2] - R[0][0] - R[1][1]) * 2.0;
        w = (R[1][0] - R[0][1]) / S; x = (R[0][2] + R[2][0]) / S; y = (R[1][2] + R[2][1]) / S; z = 0.25 * S;
    }
    const double n = std::sqrt(x * x + y * y + z * z + w * w);
    double s = 1.0 / n;
    if (w < 0.0 || (w == 0.0 && (x < 0.0 || (x == 0.0 && (y < 0.0 || (y == 0.0 && z < 0.0)))))) s = -s;
    q[0] = x * s; q[1] = y * s; q[2] = z * s; q[3] = w * s;
}

int blocks_of(long long n) { return static_cast<int>((n + SPHK_BLOCK - 1) / SPHK_BLOCK); }

// (key, value) pairs of one bin -> sorted items and cell ranges
template <int MODE>
int build_bin(sphk_mesh* m, int cells, int** start, int** items) {
    cudaStream_t st = m->stream;
    const MeshDev d = dev_of(m);
    const int nt = m->nt;
    long long *counts = nullptr, *offsets = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&counts, sizeof(long long) * (nt + 1), st));
    SPHK_CUDA_TRY(cudaMallocAsync(&offsets, sizeof(long long) * (nt + 1), st));
    k_bin_count<MODE><<<blocks_of(nt), SPHK_BLOCK, 0, st>>>(d, nt, counts);
    SPHK_CUDA_TRY(cudaMemsetAsync(counts + nt, 0, sizeof(long long), st));
    size_t tb = 0;
    SPHK_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, counts, offsets, nt + 1, st));
    void* temp = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&temp, tb, st));
    SPHK_CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, tb, counts, offsets, nt + 1, st));
    long long total = 0;
    SPHK_CUDA_TRY(cudaMemcpyAsync(&total, offsets + nt, sizeof(long long), cudaMemcpyDeviceToHost, st));
    SPHK_CUDA_TRY(cudaStreamSynchronize(st));
    SPHK_CUDA_TRY(cudaFreeAsync(temp, st));
    if (total > 0x7fffffffLL) { cudaFreeAsync(counts, st); cudaFreeAsync(offsets, st); return SPHK_ERR_ALLOC; }
    const int n = static_cast<int>(total);
    int *keys = nullptr, *vals = nullptr, *keysS = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&keys, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&vals, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&keysS, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMalloc(items, sizeof(int) * std::max(n, 1)));
    SPHK_CUDA_TRY(cudaMalloc(start, sizeof(int) * (cells + 1)));
    k_bin_write<MODE><<<blocks_of(nt), SPHK_BLOCK, 0, st>>>(d, nt, offsets, keys, vals);
    int bits = 1;
    while ((1LL << bits) < cells) ++bits;
    tb = 0;
    SPHK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keysS, vals, *items, n, 0, bits, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&temp, tb, st));
    SPHK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(temp, tb, keys, keysS, vals, *items, n, 0, bits, st));
    k_bin_start<<<blocks_of(cells + 1LL), SPHK_BLOCK, 0, st>>>(keysS, n, cells, *start);
    SPHK_CUDA_TRY(cudaGetLastError());
    for (void* p : {static_cast<void*>(counts), static_cast<void*>(offsets), static_cast<void*>(keys), static_cast<void*>(vals),
                    static_cast<void*>(keysS), temp})
        SPHK_CUDA_TRY(cudaFreeAsync(p, st));
    SPHK_CUDA_TRY(cudaStreamSynchronize(st));
    return SPHK_OK;
}

// exclusive scan of int flags -> offsets and the total (synchronises)
int scan_flags(const int* flags, int* offsets, int n, long long* total, cudaStream_t st) {
    size_t tb = 0;
    SPHK_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, flags, offsets, n, st));
    void* temp = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&temp, tb, st));
    SPHK_CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, tb, flags, offsets, n, st));
    int last[2] = {0, 0};
    SPHK_CUDA_TRY(cudaMemcpyAsync(&last[0], offsets + n - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    SPHK_CUDA_TRY(cudaMemcpyAsync(&last[1], flags + n - 1, sizeof(int), cudaMemcpyDeviceToHost, st));
    SPHK_CUDA_TRY(cudaFreeAsync(temp, st));
    SPHK_CUDA_TRY(cudaStreamSynchronize(st));
    *total = static_cast<long long>(last[0]) + last[1];
    return SPHK_OK;
}

}  // namespace

// ---- C-ABI ------------------------------------------------------------------------------------------------------------------------
extern "C" int sphk_mesh_transform(const float* v_in, int nv, float scale, const float t[3], float* v_out) {
    if (!v_in || !v_out || !t || nv <= 0 || !std::isfinite(scale) || !std::isfinite(t[0]) || !std::isfinite(t[1]) ||
        !std::isfinite(t[2]) || overlap(v_in, 12ull * nv, v_out, 12ull * nv) || overlap(t, 12, v_out, 12ull * nv))
        return SPHK_ERR_INVALID;
    for (long long i = 0; i < 3LL * nv; ++i) {
        volatile float p = scale * v_in[i];       // the product rounded to float before the add: never contracted
        v_out[i] = p + t[i % 3];
    }
    return SPHK_OK;
}

extern "C" int sphk_mesh_properties(const float* v, int nv, const int* tri, int nt, double out[SPHK_MESH_PROPS], int* flags) {
    if (!out || !flags) return SPHK_ERR_INVALID;
    const int rc = mesh_check(v, nv, tri, nt);
    if (rc != SPHK_OK) return rc;
    const bool closed = mesh_closed(tri, nt);
    std::fill(out, out + SPHK_MESH_PROPS, 0.0);
    // about the first vertex (less cancellation than about the world origin)
    const double o[3] = {v[0], v[1], v[2]};
    double area = 0.0, vol = 0.0, m1[3] = {0, 0, 0}, m2[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int t = 0; t < nt; ++t) {
        // canonical vertex order (smallest index first, then ascending) and the sign of the permutation: a reversed triangle
        // contributes exactly the negated terms, so a reversed mesh gives the same bits
        int id[3] = {tri[3 * t], tri[3 * t + 1], tri[3 * t + 2]};
        while (id[0] > id[1] || id[0] > id[2]) std::rotate(id, id + 1, id + 3);
        double sg = 1.0;
        if (id[1] > id[2]) { std::swap(id[1], id[2]); sg = -1.0; }
        double P[3][3];
        for (int k = 0; k < 3; ++k)
            for (int a = 0; a < 3; ++a) P[k][a] = static_cast<double>(v[3 * id[k] + a]) - o[a];
        const double u[3] = {P[1][0] - P[0][0], P[1][1] - P[0][1], P[1][2] - P[0][2]};
        const double w[3] = {P[2][0] - P[0][0], P[2][1] - P[0][1], P[2][2] - P[0][2]};
        const double n[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
        area += 0.5 * std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
        // tetrahedron (0, a, b, c): D = det[a, b, c]; V = D/6, int x = D/24 s, int x_i x_j = D/120 (s_i s_j + sum_p a_pi a_pj)
        const double D = sg * (P[0][0] * (P[1][1] * P[2][2] - P[1][2] * P[2][1]) - P[0][1] * (P[1][0] * P[2][2] - P[1][2] * P[2][0]) +
                               P[0][2] * (P[1][0] * P[2][1] - P[1][1] * P[2][0]));
        const double s[3] = {P[0][0] + P[1][0] + P[2][0], P[0][1] + P[1][1] + P[2][1], P[0][2] + P[1][2] + P[2][2]};
        vol += D / 6.0;
        for (int i = 0; i < 3; ++i) {
            m1[i] += D / 24.0 * s[i];
            for (int j = 0; j < 3; ++j) m2[i][j] += D / 120.0 * (s[i] * s[j] + P[0][i] * P[0][j] + P[1][i] * P[1][j] + P[2][i] * P[2][j]);
        }
    }
    out[0] = area;
    *flags = closed ? SPHK_MESH_CLOSED : 0;
    if (!closed) return SPHK_OK;
    if (!(vol != 0.0)) return SPHK_ERR_INVALID;
    const double sg = vol < 0.0 ? -1.0 : 1.0;      // reversed winding: every integral changes sign
    vol *= sg;
    double c[3], C[3][3];
    for (int i = 0; i < 3; ++i) c[i] = sg * m1[i] / vol;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[i][j] = sg * m2[i][j] - vol * c[i] * c[j];
    const double tr = C[0][0] + C[1][1] + C[2][2];
    double I[3][3];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) I[i][j] = (i == j ? tr : 0.0) - C[i][j];
    out[1] = vol;
    for (int i = 0; i < 3; ++i) out[2 + i] = c[i] + o[i];
    out[5] = I[0][0]; out[6] = I[1][1]; out[7] = I[2][2]; out[8] = I[0][1]; out[9] = I[0][2]; out[10] = I[1][2];
    double A[3][3], V[3][3];
    std::memcpy(A, I, sizeof A);
    jacobi3(A, V);
    int ord[3] = {0, 1, 2};
    std::stable_sort(ord, ord + 3, [&](int a, int b) { return A[a][a] < A[b][b]; });
    double R[3][3];
    for (int col = 0; col < 2; ++col) {
        const int e = ord[col];
        int big = 0;
        for (int k = 1; k < 3; ++k)
            if (std::fabs(V[k][e]) > std::fabs(V[big][e])) big = k;
        const double s = V[big][e] < 0.0 ? -1.0 : 1.0;
        for (int k = 0; k < 3; ++k) R[k][col] = s * V[k][e];
    }
    R[0][2] = R[1][0] * R[2][1] - R[2][0] * R[1][1];
    R[1][2] = R[2][0] * R[0][1] - R[0][0] * R[2][1];
    R[2][2] = R[0][0] * R[1][1] - R[1][0] * R[0][1];
    for (int k = 0; k < 3; ++k) out[11 + k] = A[ord[k]][ord[k]];
    quat_of(R, out + 14);
    return SPHK_OK;
}

extern "C" int sphk_mesh_create(sphk_mesh** mp, const float* v_host, int nv, const int* tri_host, int nt, void* stream) {
    if (!mp) return SPHK_ERR_INVALID;
    *mp = nullptr;
    const int rc = mesh_check(v_host, nv, tri_host, nt);
    if (rc != SPHK_OK) return rc;
    auto* m = new sphk_mesh;
    m->nv = nv; m->nt = nt; m->closed = mesh_closed(tri_host, nt) ? 1 : 0;
    m->stream = static_cast<cudaStream_t>(stream);
    double side = 0.0;
    for (int a = 0; a < 3; ++a) { m->lo[a] = v_host[a]; m->hi[a] = v_host[a]; }
    for (int i = 0; i < nv; ++i)
        for (int a = 0; a < 3; ++a) { m->lo[a] = std::min(m->lo[a], v_host[3 * i + a]); m->hi[a] = std::max(m->hi[a], v_host[3 * i + a]); }
    for (int t = 0; t < nt; ++t)
        for (int a = 0; a < 3; ++a) {
            float l = v_host[3 * tri_host[3 * t] + a], h = l;
            for (int k = 1; k < 3; ++k) { l = std::min(l, v_host[3 * tri_host[3 * t + k] + a]); h = std::max(h, v_host[3 * tri_host[3 * t + k] + a]); }
            side += (static_cast<double>(h) - l) / 3.0;
        }
    side /= nt;                                   // mean bounding-box side of a triangle
    const double e[3] = {static_cast<double>(m->hi[0]) - m->lo[0], static_cast<double>(m->hi[1]) - m->lo[1],
                         static_cast<double>(m->hi[2]) - m->lo[2]};
    const double emax = std::max({e[0], e[1], e[2]});
    // at most 128 cells per axis in 3D and 512 columns per axis in (x, z), and no cell smaller than a typical triangle
    m->h3 = static_cast<float>(std::max({emax / 128.0, side, 1e-30}));
    m->h2 = static_cast<float>(std::max({std::max(e[0], e[2]) / 512.0, side, 1e-30}));
    m->inv3 = 1.0f / m->h3;
    m->inv2 = 1.0f / m->h2;
    for (int a = 0; a < 3; ++a) m->d3[a] = std::min(1 + static_cast<int>(std::floor(e[a] * m->inv3)), 129);
    m->d2[0] = std::min(1 + static_cast<int>(std::floor(e[0] * m->inv2)), 513);
    m->d2[1] = std::min(1 + static_cast<int>(std::floor(e[2] * m->inv2)), 513);
    int r = SPHK_OK;
    if (cudaMalloc(&m->v, sizeof(float) * 3 * nv) != cudaSuccess || cudaMalloc(&m->tri, sizeof(int) * 3 * nt) != cudaSuccess) r = SPHK_ERR_ALLOC;
    if (r == SPHK_OK && (cudaMemcpyAsync(m->v, v_host, sizeof(float) * 3 * nv, cudaMemcpyHostToDevice, m->stream) != cudaSuccess ||
                         cudaMemcpyAsync(m->tri, tri_host, sizeof(int) * 3 * nt, cudaMemcpyHostToDevice, m->stream) != cudaSuccess))
        r = SPHK_ERR_ALLOC;
    if (r == SPHK_OK) r = build_bin<3>(m, m->d3[0] * m->d3[1] * m->d3[2], &m->start3, &m->items3);
    if (r == SPHK_OK) r = build_bin<2>(m, m->d2[0] * m->d2[1], &m->start2, &m->items2);
    if (r != SPHK_OK) { sphk_mesh_destroy(m); return r; }
    *mp = m;
    return SPHK_OK;
}

extern "C" void sphk_mesh_destroy(sphk_mesh* m) {
    if (!m) return;
    if (m->stream) cudaStreamSynchronize(m->stream);
    cudaFree(m->v); cudaFree(m->tri); cudaFree(m->start3); cudaFree(m->items3); cudaFree(m->start2); cudaFree(m->items2);
    delete m;
}

extern "C" int sphk_mesh_classify(const sphk_mesh* m, const float* pos, int n, float clearance, int* flags_out) {
    if (!m || !pos || !flags_out || n <= 0 || !m->closed || !(clearance >= 0.0f) || !std::isfinite(clearance) ||
        overlap(pos, 12ull * n, flags_out, 4ull * n))
        return SPHK_ERR_INVALID;
    k_mesh_classify<<<blocks_of(n), SPHK_BLOCK, 0, m->stream>>>(dev_of(m), pos, n, clearance, flags_out);
    SPHK_CUDA_TRY(cudaGetLastError());
    return SPHK_OK;
}

extern "C" int sphk_mesh_fill(const sphk_mesh* m, float spacing, const float origin[3], float clearance, float* pos_out, int capacity,
                              int* count_host) {
    if (!m || !origin || !pos_out || !count_host || !m->closed || !(spacing > 0.0f) || !std::isfinite(spacing) ||
        !(clearance >= 0.0f) || !std::isfinite(clearance) || capacity < 0 || !std::isfinite(origin[0]) || !std::isfinite(origin[1]) ||
        !std::isfinite(origin[2]) || overlap(count_host, 4, pos_out, 12ull * capacity))
        return SPHK_ERR_INVALID;
    // index ranges over the bounding box, one index of margin on each side (those points are outside)
    long long r0[3], r1[3];
    for (int a = 0; a < 3; ++a) {
        r0[a] = static_cast<long long>(std::floor((static_cast<double>(m->lo[a]) - origin[a]) / spacing)) - 1;
        r1[a] = static_cast<long long>(std::floor((static_cast<double>(m->hi[a]) - origin[a]) / spacing)) + 1;
        if (r0[a] < -(1LL << 24) || r1[a] > (1LL << 24)) return SPHK_ERR_INVALID;   // indices exact in float
    }
    const long long total = (r1[0] - r0[0] + 1) * (r1[1] - r0[1] + 1) * (r1[2] - r0[2] + 1);
    if (total > 0x7fffffffLL) return SPHK_ERR_INVALID;
    Lattice L{origin[0], origin[1], origin[2], spacing, static_cast<int>(r0[0]), static_cast<int>(r0[1]), static_cast<int>(r0[2]),
              static_cast<int>(r1[0] - r0[0] + 1), static_cast<int>(r1[1] - r0[1] + 1), static_cast<int>(r1[2] - r0[2] + 1)};
    const int n = static_cast<int>(total);
    cudaStream_t st = m->stream;
    int *keep = nullptr, *offset = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&keep, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&offset, sizeof(int) * n, st));
    k_fill_flag<<<blocks_of(n), SPHK_BLOCK, 0, st>>>(dev_of(m), L, n, clearance, keep);
    SPHK_CUDA_TRY(cudaGetLastError());
    long long count = 0;
    int rc = scan_flags(keep, offset, n, &count, st);
    if (rc == SPHK_OK && count <= capacity) {
        k_fill_write<<<blocks_of(n), SPHK_BLOCK, 0, st>>>(L, n, keep, offset, pos_out);
        rc = cudaGetLastError() == cudaSuccess ? SPHK_OK : SPHK_ERR_ALLOC;
    }
    cudaFreeAsync(keep, st);
    cudaFreeAsync(offset, st);
    SPHK_CUDA_TRY(cudaStreamSynchronize(st));
    *count_host = static_cast<int>(count);
    return rc;
}

extern "C" int sphk_mesh_sample_surface(const sphk_mesh* m, float r, float* pos_out, int capacity, int* count_host) {
    if (!m || !pos_out || !count_host || !(r > 0.0f) || !std::isfinite(r) || capacity < 0 || overlap(count_host, 4, pos_out, 12ull * capacity))
        return SPHK_ERR_INVALID;
    cudaStream_t st = m->stream;
    const int nt = m->nt;
    const float step = 0.25f * r;
    long long *counts = nullptr, *offsets = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&counts, sizeof(long long) * (nt + 1), st));
    SPHK_CUDA_TRY(cudaMallocAsync(&offsets, sizeof(long long) * (nt + 1), st));
    k_cand_count<<<blocks_of(nt), SPHK_BLOCK, 0, st>>>(m->v, m->tri, nt, step, counts);
    SPHK_CUDA_TRY(cudaMemsetAsync(counts + nt, 0, sizeof(long long), st));
    size_t tb = 0;
    SPHK_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, counts, offsets, nt + 1, st));
    void* temp = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&temp, tb, st));
    SPHK_CUDA_TRY(cub::DeviceScan::ExclusiveSum(temp, tb, counts, offsets, nt + 1, st));
    SPHK_CUDA_TRY(cudaFreeAsync(temp, st));
    long long total = 0;
    SPHK_CUDA_TRY(cudaMemcpyAsync(&total, offsets + nt, sizeof(long long), cudaMemcpyDeviceToHost, st));
    SPHK_CUDA_TRY(cudaStreamSynchronize(st));
    if (total > 0x7fffffffLL) { cudaFreeAsync(counts, st); cudaFreeAsync(offsets, st); cudaStreamSynchronize(st); return SPHK_ERR_INVALID; }
    const int n = static_cast<int>(total);
    // cells of side r (1 + 1e-5): two points two cells apart are farther than r even after the rounding of their cell index
    const double side = static_cast<double>(r) * (1.0 + 1e-5);
    SampleGrid g{m->lo[0], m->lo[1], m->lo[2], static_cast<float>(1.0 / side), 0, 0, 0};
    g.dx = 1 + static_cast<long long>((static_cast<double>(m->hi[0]) - m->lo[0]) / side);
    g.dy = 1 + static_cast<long long>((static_cast<double>(m->hi[1]) - m->lo[1]) / side);
    g.dz = 1 + static_cast<long long>((static_cast<double>(m->hi[2]) - m->lo[2]) / side);
    float* cand = nullptr;
    unsigned long long *keys = nullptr, *keysS = nullptr, *cellKey = nullptr;
    int *idx = nullptr, *idxS = nullptr, *head = nullptr, *cellOf = nullptr, *cellStart = nullptr, *accCount = nullptr,
        *accepted = nullptr, *offset = nullptr, *overflow = nullptr;
    float3* acc = nullptr;
    SPHK_CUDA_TRY(cudaMallocAsync(&cand, sizeof(float) * 3 * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&keys, sizeof(unsigned long long) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&keysS, sizeof(unsigned long long) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&idx, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&idxS, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&head, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&cellOf, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&accepted, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&offset, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&overflow, sizeof(int), st));
    k_cand_write<<<blocks_of(nt), SPHK_BLOCK, 0, st>>>(m->v, m->tri, nt, step, g, offsets, cand, keys, idx);
    const unsigned long long cells = static_cast<unsigned long long>(g.dx) * g.dy * g.dz;
    int bits = 1;
    while (bits < 64 && (1ULL << bits) < cells) ++bits;
    tb = 0;
    SPHK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, keysS, idx, idxS, n, 0, bits, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&temp, tb, st));
    SPHK_CUDA_TRY(cub::DeviceRadixSort::SortPairs(temp, tb, keys, keysS, idx, idxS, n, 0, bits, st));
    SPHK_CUDA_TRY(cudaFreeAsync(temp, st));
    k_cell_heads<<<blocks_of(n), SPHK_BLOCK, 0, st>>>(keysS, n, head);
    long long nCellsLL = 0;
    int rc = scan_flags(head, cellOf, n, &nCellsLL, st);
    if (rc != SPHK_OK) return rc;
    const int nCells = static_cast<int>(nCellsLL);
    SPHK_CUDA_TRY(cudaMallocAsync(&cellKey, sizeof(unsigned long long) * nCells, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&cellStart, sizeof(int) * (nCells + 1), st));
    SPHK_CUDA_TRY(cudaMallocAsync(&accCount, sizeof(int) * nCells, st));
    SPHK_CUDA_TRY(cudaMallocAsync(&acc, sizeof(float3) * kCellSamples * nCells, st));
    k_cell_list<<<blocks_of(n), SPHK_BLOCK, 0, st>>>(keysS, n, head, cellOf, cellKey, cellStart);
    SPHK_CUDA_TRY(cudaMemcpyAsync(cellStart + nCells, &n, sizeof(int), cudaMemcpyHostToDevice, st));
    SPHK_CUDA_TRY(cudaMemsetAsync(accCount, 0, sizeof(int) * nCells, st));
    SPHK_CUDA_TRY(cudaMemsetAsync(accepted, 0, sizeof(int) * n, st));
    SPHK_CUDA_TRY(cudaMemsetAsync(overflow, 0, sizeof(int), st));
    const double rr = static_cast<double>(r) * r;
    for (int phase = 0; phase < 27; ++phase)
        k_sample_phase<<<blocks_of(nCells), SPHK_BLOCK, 0, st>>>(g, phase, cellKey, cellStart, nCells, idxS, cand, rr, acc, accCount,
                                                                 accepted, overflow);
    SPHK_CUDA_TRY(cudaGetLastError());
    long long count = 0;
    rc = scan_flags(accepted, offset, n, &count, st);
    int over = 0;
    if (rc == SPHK_OK) rc = cudaMemcpy(&over, overflow, sizeof(int), cudaMemcpyDeviceToHost) == cudaSuccess ? SPHK_OK : SPHK_ERR_ALLOC;
    if (rc == SPHK_OK && over) rc = SPHK_ERR_CAPACITY;
    if (rc == SPHK_OK && count <= capacity) {
        k_sample_write<<<blocks_of(n), SPHK_BLOCK, 0, st>>>(n, accepted, offset, idxS, cand, pos_out);
        rc = cudaGetLastError() == cudaSuccess ? SPHK_OK : SPHK_ERR_ALLOC;
    }
    for (void* p : {static_cast<void*>(counts), static_cast<void*>(offsets), static_cast<void*>(cand), static_cast<void*>(keys),
                    static_cast<void*>(keysS), static_cast<void*>(idx), static_cast<void*>(idxS), static_cast<void*>(head),
                    static_cast<void*>(cellOf), static_cast<void*>(accepted), static_cast<void*>(offset), static_cast<void*>(overflow),
                    static_cast<void*>(cellKey), static_cast<void*>(cellStart), static_cast<void*>(accCount), static_cast<void*>(acc)})
        cudaFreeAsync(p, st);
    SPHK_CUDA_TRY(cudaStreamSynchronize(st));
    *count_host = static_cast<int>(count);
    return rc;
}
