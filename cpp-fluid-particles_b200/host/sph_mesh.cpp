// sph_mesh.cpp -- scenes from triangle meshes in the class layer (DESIGN.md section 2.12): the OBJ reader and thin wrappers of the
// sphk_mesh_* entries of the C-ABI that build point sets and bodies.  No device code here: this file is compiled by g++.
#include "sph_api.hpp"

#include <cerrno>
#include <cmath>
#include <cstdlib>
#include <fstream>
#include <sstream>
#include <stdexcept>

namespace sphb200 {
namespace {

[[noreturn]] void fail(const std::string& what) { throw std::runtime_error(what); }

void ok(int rc, const char* what) {
    if (rc != 0) fail(std::string(what) + ": " + sphk_error_string(rc) + " (" + std::to_string(rc) + ")");
}

// a device mesh for the lifetime of one call
struct DeviceMesh {
    sphk_mesh* m = nullptr;
    explicit DeviceMesh(const TriangleMesh& mesh) {
        ok(sphk_mesh_create(&m, reinterpret_cast<const float*>(mesh.vertices.data()), static_cast<int>(mesh.vertices.size()),
                            reinterpret_cast<const int*>(mesh.triangles.data()), static_cast<int>(mesh.triangles.size()), nullptr),
           "sphk_mesh_create");
    }
    ~DeviceMesh() { sphk_mesh_destroy(m); }
};

struct DeviceBuffer {
    void* p = nullptr;
    explicit DeviceBuffer(size_t bytes) {
        if (cudaMalloc(&p, std::max<size_t>(bytes, 4)) != cudaSuccess) fail("cudaMalloc of " + std::to_string(bytes) + " bytes failed");
    }
    ~DeviceBuffer() { cudaFree(p); }
};

std::vector<float3> download(const DeviceBuffer& b, int n) {
    std::vector<float3> out(static_cast<size_t>(n));
    if (n > 0 && cudaMemcpy(out.data(), b.p, sizeof(float3) * n, cudaMemcpyDeviceToHost) != cudaSuccess) fail("cudaMemcpy failed");
    return out;
}

// runs `call(buffer, capacity, &count)` with an estimated capacity, and once more with the exact one when that was too small
template <class F>
std::vector<float3> counted(long long estimate, F call) {
    int cap = static_cast<int>(std::min<long long>(std::max<long long>(estimate, 1024), 0x7fffffffLL / 12));
    for (;;) {
        DeviceBuffer b(sizeof(float3) * static_cast<size_t>(cap));
        int count = 0;
        call(static_cast<float*>(b.p), cap, &count);
        if (count <= cap) return download(b, count);
        cap = count;
    }
}

bool number(const std::string& tok, float& x) {
    char* end = nullptr;
    errno = 0;
    x = std::strtof(tok.c_str(), &end);
    return !tok.empty() && *end == '\0' && errno != ERANGE && std::isfinite(x);
}

}  // namespace

TriangleMesh loadObj(const std::string& path, float scale, float3 translate) {
    std::ifstream in(path);
    if (!in) fail(path + ": cannot open");
    std::vector<float> v;
    std::vector<int> tri;
    std::vector<long long> faceLine;          // the line of every triangle, for the index check after the last vertex
    std::string line;
    long long lineNo = 0;
    while (std::getline(in, line)) {
        ++lineNo;
        const size_t hash = line.find('#');
        if (hash != std::string::npos) line.resize(hash);
        std::istringstream ss(line);
        std::string key, tok;
        if (!(ss >> key)) continue;
        const std::string where = path + ":" + std::to_string(lineNo) + ": ";
        if (key == "v") {
            std::vector<float> xs;
            while (ss >> tok) {
                float x;
                if (!number(tok, x)) fail(where + "bad number '" + tok + "'");
                xs.push_back(x);
            }
            if (xs.size() != 3 && xs.size() != 4) fail(where + "a vertex needs x y z [w]");
            v.insert(v.end(), xs.begin(), xs.begin() + 3);
        } else if (key == "f") {
            std::vector<int> idx;
            while (ss >> tok) {
                const std::string head = tok.substr(0, tok.find('/'));
                char* end = nullptr;
                errno = 0;
                const long k = std::strtol(head.c_str(), &end, 10);
                const long nv = static_cast<long>(v.size() / 3);
                if (head.empty() || *end != '\0' || errno == ERANGE || k == 0 || k > 0x7fffffffL || (k < 0 && -k > nv))
                    fail(where + "bad vertex index '" + tok + "'");
                idx.push_back(static_cast<int>(k > 0 ? k - 1 : nv + k));
            }
            if (idx.size() < 3) fail(where + "a face needs at least 3 vertices");
            for (size_t k = 1; k + 1 < idx.size(); ++k) {
                tri.insert(tri.end(), {idx[0], idx[k], idx[k + 1]});
                faceLine.push_back(lineNo);
            }
        }
    }
    const long long nv = static_cast<long long>(v.size() / 3);
    for (size_t t = 0; t < faceLine.size(); ++t)
        for (int k = 0; k < 3; ++k)
            if (tri[3 * t + k] >= nv)
                fail(path + ":" + std::to_string(faceLine[t]) + ": vertex index " + std::to_string(tri[3 * t + k] + 1) + " beyond the " +
                     std::to_string(nv) + " vertices");
    if (nv == 0 || tri.empty()) fail(path + ": no vertices or no faces");
    TriangleMesh m;
    m.vertices.resize(static_cast<size_t>(nv));
    const float t[3] = {translate.x, translate.y, translate.z};
    ok(sphk_mesh_transform(v.data(), static_cast<int>(nv), scale, t, reinterpret_cast<float*>(m.vertices.data())), "sphk_mesh_transform");
    m.triangles.resize(tri.size() / 3);
    for (size_t k = 0; k < m.triangles.size(); ++k) m.triangles[k] = int3{tri[3 * k], tri[3 * k + 1], tri[3 * k + 2]};
    return m;
}

MeshProperties meshProperties(const TriangleMesh& mesh) {
    double out[SPHK_MESH_PROPS];
    int flags = 0;
    ok(sphk_mesh_properties(reinterpret_cast<const float*>(mesh.vertices.data()), static_cast<int>(mesh.vertices.size()),
                            reinterpret_cast<const int*>(mesh.triangles.data()), static_cast<int>(mesh.triangles.size()), out, &flags),
       "sphk_mesh_properties");
    MeshProperties p;
    p.closed = (flags & SPHK_MESH_CLOSED) != 0;
    p.area = out[0];
    p.volume = out[1];
    std::copy(out + 2, out + 5, p.centroid);
    std::copy(out + 5, out + 11, p.inertia);
    std::copy(out + 11, out + 14, p.principal);
    if (p.closed) std::copy(out + 14, out + 18, p.orientation);
    return p;
}

std::vector<float3> sampleSurface(const TriangleMesh& mesh, float r) {
    const MeshProperties p = meshProperties(mesh);
    const DeviceMesh d(mesh);
    // a plane holds at most 2 / (sqrt(3) r^2) samples per unit area
    return counted(static_cast<long long>(1.3 * p.area / (double(r) * r)) + 64,
                   [&](float* out, int cap, int* n) { ok(sphk_mesh_sample_surface(d.m, r, out, cap, n), "sphk_mesh_sample_surface"); });
}

std::vector<float3> fillMesh(const TriangleMesh& mesh, float spacing, float3 origin, float clearance) {
    const MeshProperties p = meshProperties(mesh);
    const DeviceMesh d(mesh);
    const float o[3] = {origin.x, origin.y, origin.z};
    return counted(static_cast<long long>(1.1 * p.volume / (double(spacing) * spacing * spacing)) + 64,
                   [&](float* out, int cap, int* n) { ok(sphk_mesh_fill(d.m, spacing, o, clearance, out, cap, n), "sphk_mesh_fill"); });
}

std::vector<float3> clearOf(const std::vector<float3>& points, const std::vector<TriangleMesh>& meshes, float clearance) {
    if (points.empty() || meshes.empty()) return points;
    const int n = static_cast<int>(points.size());
    DeviceBuffer pos(sizeof(float3) * points.size()), flags(sizeof(int) * points.size());
    if (cudaMemcpy(pos.p, points.data(), sizeof(float3) * points.size(), cudaMemcpyHostToDevice) != cudaSuccess) fail("cudaMemcpy failed");
    std::vector<int> f(points.size()), drop(points.size(), 0);
    for (const TriangleMesh& mesh : meshes) {
        const DeviceMesh d(mesh);
        ok(sphk_mesh_classify(d.m, static_cast<const float*>(pos.p), n, clearance, static_cast<int*>(flags.p)), "sphk_mesh_classify");
        if (cudaMemcpy(f.data(), flags.p, sizeof(int) * points.size(), cudaMemcpyDeviceToHost) != cudaSuccess) fail("cudaMemcpy failed");
        for (size_t i = 0; i < f.size(); ++i) drop[i] |= f[i];
    }
    std::vector<float3> out;
    for (size_t i = 0; i < points.size(); ++i)
        if (!drop[i]) out.push_back(points[i]);
    return out;
}

KinematicBody meshBody(const TriangleMesh& mesh, float r, float relDensity, float fluidMassPerVolume) {
    const MeshProperties p = meshProperties(mesh);
    if (!p.closed) fail("meshBody: the mesh is not closed");
    if (!(relDensity >= 0.0f) || !std::isfinite(relDensity)) fail("meshBody: the relative density must be finite and >= 0");
    const double x = p.orientation[0], y = p.orientation[1], z = p.orientation[2], w = p.orientation[3];
    // R(q): body -> world; a body point is R^T (p - c), every operation in double in this order (meshes.py repeats it)
    const double R[3][3] = {{1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - z * w), 2.0 * (x * z + y * w)},
                            {2.0 * (x * y + z * w), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - x * w)},
                            {2.0 * (x * z - y * w), 2.0 * (y * z + x * w), 1.0 - 2.0 * (x * x + y * y)}};
    KinematicBody b;
    for (const float3& s : sampleSurface(mesh, r)) {
        const double d[3] = {double(s.x) - p.centroid[0], double(s.y) - p.centroid[1], double(s.z) - p.centroid[2]};
        float l[3];
        for (int k = 0; k < 3; ++k) l[k] = static_cast<float>(R[0][k] * d[0] + R[1][k] * d[1] + R[2][k] * d[2]);
        b.points.push_back(make_float3(l[0], l[1], l[2]));
    }
    b.position = make_float3(float(p.centroid[0]), float(p.centroid[1]), float(p.centroid[2]));
    b.orientation = make_float4(float(x), float(y), float(z), float(w));
    b.linearVelocity = make_float3(0.0f, 0.0f, 0.0f);
    b.angularVelocity = make_float3(0.0f, 0.0f, 0.0f);
    const double rho = double(relDensity) * double(fluidMassPerVolume);
    b.mass = static_cast<float>(rho * p.volume);
    b.inertia = make_float3(float(p.principal[0] * rho), float(p.principal[1] * rho), float(p.principal[2] * rho));
    return b;
}

}  // namespace sphb200
