// sphk_state.cu -- checkpoints: the file format, the pack kernel with its checksums, the asynchronous save and the verified load
// (sphk.h, "checkpoints"; DESIGN.md section 2.14).  The only module that knows the format.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "sphk_internal.cuh"

static_assert(sizeof(sphk_state_config) == 152, "sphk_state_config is part of the file format");

namespace {
constexpr char kMagic[8] = {'S', 'P', 'H', 'K', 'C', 'K', 'P', 'T'};
constexpr unsigned long long kGamma = 0x9E3779B97F4A7C15ull;
constexpr int kPackThreads = 256, kPackUnits = 8;          // a block packs 256 x 8 units of 16 bytes (32 KiB)
constexpr unsigned long long kBlockBytes = 16ull * kPackThreads * kPackUnits;
constexpr size_t kFixed = 40 + sizeof(sphk_state_config); // magic .. config
constexpr size_t kEntry = 64;                             // one section-table entry

__host__ __device__ __forceinline__ unsigned long long splitmix(unsigned long long z) {
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

struct PackEntry {
    const unsigned char* src;
    unsigned char* dst;              // 16-byte aligned staging slot, or nullptr: checksum only
    unsigned long long bytes;
    unsigned long long blockBegin;   // first block of this entry
};

// One launch over every section: block b packs 32 KiB of the entry whose blocks contain b (16-byte loads where the source is
// aligned, the zero-padded tail byte by byte) and adds its share of the entry's checksum.  The sum is order-independent, so the
// integer atomics give the same value every time.
__global__ void __launch_bounds__(kPackThreads) k_state_pack(const PackEntry* __restrict__ table, int n, unsigned long long* __restrict__ sums) {
    __shared__ int sec;
    __shared__ unsigned long long part[kPackThreads / 32];
    if (threadIdx.x == 0) {
        int s = 0;
        while (s + 1 < n && table[s + 1].blockBegin <= blockIdx.x) ++s;
        sec = s;
    }
    __syncthreads();
    const PackEntry e = table[sec];
    const unsigned long long units = (e.bytes + 15) / 16, words = (e.bytes + 7) / 8;
    const bool vec = (reinterpret_cast<uintptr_t>(e.src) & 15) == 0;
    const unsigned long long first = (blockIdx.x - e.blockBegin) * static_cast<unsigned long long>(kPackThreads * kPackUnits);
    unsigned long long acc = 0;
#pragma unroll
    for (int k = 0; k < kPackUnits; ++k) {
        const unsigned long long u = first + static_cast<unsigned long long>(k) * kPackThreads + threadIdx.x;
        if (u >= units) break;
        uint4 v;
        if (vec && (u + 1) * 16 <= e.bytes) {
            v = __ldg(reinterpret_cast<const uint4*>(e.src) + u);
        } else {
            unsigned int w[4] = {0, 0, 0, 0};
            for (int i = 0; i < 16; ++i) {
                const unsigned long long at = u * 16 + i;
                if (at < e.bytes) w[i / 4] |= static_cast<unsigned int>(e.src[at]) << (8 * (i % 4));
            }
            v = make_uint4(w[0], w[1], w[2], w[3]);
        }
        if (e.dst) reinterpret_cast<uint4*>(e.dst)[u] = v;
        const unsigned long long w0 = v.x | (static_cast<unsigned long long>(v.y) << 32);
        const unsigned long long w1 = v.z | (static_cast<unsigned long long>(v.w) << 32);
        if (2 * u < words) acc += splitmix(w0 + (2 * u + 1) * kGamma);
        if (2 * u + 1 < words) acc += splitmix(w1 + (2 * u + 2) * kGamma);
    }
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x / 32] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < kPackThreads / 32; ++w) t += part[w];
        atomicAdd(sums + sec, t);
    }
}

unsigned long long align16(unsigned long long x) { return (x + 15) & ~15ull; }

void say(char* msg, int len, const char* fmt, ...) {
    if (!msg || len <= 0) return;
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(msg, static_cast<size_t>(len), fmt, ap);
    va_end(ap);
}

struct CrcTable {
    unsigned int t[256];
};

unsigned int crc32(const unsigned char* p, size_t n) {
    // built once, thread-safely (the writer threads and a restore may run this at the same time)
    static const CrcTable table = [] {
        CrcTable r{};
        for (unsigned int i = 0; i < 256; ++i) {
            unsigned int c = i;
            for (int k = 0; k < 8; ++k) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            r.t[i] = c;
        }
        return r;
    }();
    unsigned int c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) c = table.t[(c ^ p[i]) & 0xFF] ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

unsigned long long checksum_host(const unsigned char* p, unsigned long long bytes) {
    unsigned long long h = 0;
    const unsigned long long words = (bytes + 7) / 8;
    for (unsigned long long i = 0; i < words; ++i) {
        unsigned long long w = 0;
        const unsigned long long k = bytes - 8 * i < 8 ? bytes - 8 * i : 8;
        std::memcpy(&w, p + 8 * i, static_cast<size_t>(k));      // little-endian hosts only (x86-64, aarch64)
        h += splitmix(w + (i + 1) * kGamma);
    }
    return h;
}

// the section table as it goes into the file
struct Entry {
    char name[SPHK_STATE_NAME];
    unsigned long long offset, bytes;
    unsigned int elem;
    unsigned int host;
    unsigned long long sum;
};
static_assert(sizeof(Entry) == kEntry, "section-table entry is part of the file format");

size_t header_bytes(int n) { return static_cast<size_t>(align16(kFixed + kEntry * n + 8)); }

std::vector<unsigned char> make_header(const sphk_state_config& cfg, const std::vector<Entry>& table, unsigned long long fileBytes) {
    const int n = static_cast<int>(table.size());
    std::vector<unsigned char> h(header_bytes(n), 0);
    const unsigned int version = SPHK_STATE_VERSION, sections = static_cast<unsigned int>(n);
    const unsigned long long hb = h.size(), cfgHash = checksum_host(reinterpret_cast<const unsigned char*>(&cfg), sizeof(cfg));
    std::memcpy(h.data(), kMagic, 8);
    std::memcpy(h.data() + 8, &version, 4);
    std::memcpy(h.data() + 12, &sections, 4);
    std::memcpy(h.data() + 16, &hb, 8);
    std::memcpy(h.data() + 24, &fileBytes, 8);
    std::memcpy(h.data() + 32, &cfgHash, 8);
    std::memcpy(h.data() + 40, &cfg, sizeof(cfg));
    if (n) std::memcpy(h.data() + kFixed, table.data(), kEntry * n);
    const unsigned int crc = crc32(h.data(), kFixed + kEntry * n);
    std::memcpy(h.data() + kFixed + kEntry * n, &crc, 4);
    return h;
}

// the context's own sections, after the caller's
void ctx_sections(const sphk_ctx* c, std::vector<sphk_state_section>& out) {
    auto add = [&](const char* name, void* p, unsigned long long bytes, unsigned int elem) {
        sphk_state_section s{};
        std::snprintf(s.name, sizeof(s.name), "%s", name);
        s.ptr = p; s.bytes = bytes; s.elem_size = elem; s.host = 0;
        out.push_back(s);
    };
    if (const BodyState* B = c->bodies) {
        add("ctx.body_pose", B->pose, 28ull * B->nBodies, 4);
        add("ctx.body_motion", B->motion, 24ull * B->nBodies, 4);
        if (B->impulse) add("ctx.body_impulse", B->impulse, 24ull * B->nBodies, 4);
        add("ctx.body_local", B->local, 16ull * B->n, 16);
        add("ctx.body_decl", B->decl, 4ull * B->n, 4);
    }
    if (c->openDev) add("ctx.open_check", c->openDev + 1, 4, 4);
}

bool valid_sections(const sphk_state_section* s, int n) {
    if (n < 0 || (n > 0 && !s)) return false;
    for (int i = 0; i < n; ++i) {
        if (s[i].bytes && !s[i].ptr) return false;
        if (std::memchr(s[i].name, 0, SPHK_STATE_NAME) == nullptr || s[i].name[0] == 0) return false;
        if (s[i].host != 0 && s[i].host != 1) return false;
    }
    return true;
}
}  // namespace

// one per context: the staging memory and the save in flight
struct StateStage {
    unsigned char* dev = nullptr; size_t devCap = 0;           // device staging of the payload
    unsigned char* pinned = nullptr; size_t pinnedCap = 0;     // its host copy
    PackEntry* table = nullptr;                                // device [SPHK_STATE_MAX_SECTIONS + 8]
    PackEntry* tableHost = nullptr;                            // pinned, the same
    unsigned long long* sums = nullptr;                        // device [SPHK_STATE_MAX_SECTIONS + 8]
    unsigned long long* sumsHost = nullptr;                    // pinned
    cudaStream_t copy = nullptr;
    cudaEvent_t packed = nullptr, copied = nullptr;
    std::thread writer;
    bool pending = false;
    int result = 0;
    std::string message;
};

struct sphk_state_file {
    std::vector<unsigned char> bytes;
    sphk_state_config config{};
    std::vector<Entry> table;
};

static int stage_init(sphk_ctx* c) {
    if (c->state) return SPHK_OK;
    StateStage* S = new StateStage();
    const size_t tb = sizeof(PackEntry) * (SPHK_STATE_MAX_SECTIONS + 8), sb = 8 * (SPHK_STATE_MAX_SECTIONS + 8);
    cudaError_t e = cudaMalloc(&S->table, tb);
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&S->tableHost), tb);
    if (e == cudaSuccess) e = cudaMalloc(&S->sums, sb);
    if (e == cudaSuccess) e = cudaMallocHost(reinterpret_cast<void**>(&S->sumsHost), sb);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&S->copy, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&S->packed, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&S->copied, cudaEventDisableTiming);
    c->state = S;
    if (e != cudaSuccess) { cudaGetLastError(); sphk_checkpoint_release(c); return SPHK_ERR_ALLOC; }
    return SPHK_OK;
}

static int stage_reserve(StateStage* S, size_t bytes, bool pinned) {
    if (bytes > S->devCap) {
        cudaFree(S->dev); S->dev = nullptr; S->devCap = 0;
        if (cudaMalloc(&S->dev, bytes) != cudaSuccess) { cudaGetLastError(); return SPHK_ERR_ALLOC; }
        S->devCap = bytes;
    }
    if (pinned && bytes > S->pinnedCap) {
        if (S->pinned) cudaFreeHost(S->pinned);
        S->pinned = nullptr; S->pinnedCap = 0;
        if (cudaMallocHost(reinterpret_cast<void**>(&S->pinned), bytes) != cudaSuccess) { cudaGetLastError(); return SPHK_ERR_ALLOC; }
        S->pinnedCap = bytes;
    }
    return SPHK_OK;
}

static void stage_join(StateStage* S) {
    if (S && S->writer.joinable()) S->writer.join();
}

// enqueues the pack of `entries` (dst set) or their checksums (dst nullptr) and the copy of the sums into sumsHost
static int enqueue_pack(sphk_ctx* c, StateStage* S, int n) {
    unsigned long long blocks = 0;
    for (int i = 0; i < n; ++i) {
        S->tableHost[i].blockBegin = blocks;
        blocks += (S->tableHost[i].bytes + kBlockBytes - 1) / kBlockBytes;
    }
    SPHK_CUDA_TRY(cudaMemcpyAsync(S->table, S->tableHost, sizeof(PackEntry) * n, cudaMemcpyHostToDevice, c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(S->sums, 0, 8ull * n, c->stream));
    if (blocks > 0x7fffffffull) return SPHK_ERR_INVALID;
    if (blocks) {
        k_state_pack<<<static_cast<unsigned int>(blocks), kPackThreads, 0, c->stream>>>(S->table, n, S->sums);
        SPHK_CUDA_TRY(cudaGetLastError());
        ++c->launches;
    }
    return SPHK_OK;
}

extern "C" int sphk_state_checksum_host(const void* data, unsigned long long bytes, unsigned long long* out) {
    if (!out || (bytes && !data)) return SPHK_ERR_INVALID;
    *out = checksum_host(static_cast<const unsigned char*>(data), bytes);
    return SPHK_OK;
}

extern "C" int sphk_state_crc32_host(const void* data, unsigned long long bytes, unsigned int* out) {
    if (!out || (bytes && !data)) return SPHK_ERR_INVALID;
    *out = crc32(static_cast<const unsigned char*>(data), static_cast<size_t>(bytes));
    return SPHK_OK;
}

extern "C" int sphk_state_checksum_device(sphk_ctx* c, const void* data, unsigned long long bytes, unsigned long long* out) {
    if (!c || !out || (bytes && !data)) return SPHK_ERR_INVALID;
    if (int rc = stage_init(c)) return rc;
    StateStage* S = c->state;
    stage_join(S);
    S->tableHost[0] = PackEntry{static_cast<const unsigned char*>(data), nullptr, bytes, 0};
    if (int rc = enqueue_pack(c, S, 1)) return rc;
    SPHK_CUDA_TRY(cudaMemcpyAsync(S->sumsHost, S->sums, 8, cudaMemcpyDeviceToHost, c->stream));
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    *out = S->sumsHost[0];
    return SPHK_OK;
}

static int write_file(const std::string& path, const std::vector<unsigned char>& header, const unsigned char* payload, size_t bytes,
                      std::string& why) {
    const std::string tmp = path + ".tmp";
    const int fd = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fd < 0) { why = "cannot create " + tmp + ": " + std::strerror(errno); return SPHK_ERR_INVALID; }
    auto put = [&](const unsigned char* p, size_t n) {
        while (n) {
            const ssize_t w = ::write(fd, p, n);
            if (w < 0) { if (errno == EINTR) continue; return false; }
            p += w; n -= static_cast<size_t>(w);
        }
        return true;
    };
    bool ok = put(header.data(), header.size()) && put(payload, bytes);
    if (!ok) why = "cannot write " + tmp + ": " + std::strerror(errno);
    if (ok && ::fsync(fd) != 0) { ok = false; why = "cannot fsync " + tmp + ": " + std::strerror(errno); }
    if (::close(fd) != 0 && ok) { ok = false; why = "cannot close " + tmp + ": " + std::strerror(errno); }
    if (ok && ::rename(tmp.c_str(), path.c_str()) != 0) { ok = false; why = "cannot rename " + tmp + ": " + std::strerror(errno); }
    if (!ok) { ::unlink(tmp.c_str()); return SPHK_ERR_INVALID; }
    // the rename itself is durable once the directory is synced
    const size_t slash = path.rfind('/');
    const std::string dir = slash == std::string::npos ? "." : (slash == 0 ? "/" : path.substr(0, slash));
    const int dfd = ::open(dir.c_str(), O_RDONLY);
    if (dfd >= 0) { ::fsync(dfd); ::close(dfd); }
    return SPHK_OK;
}

extern "C" int sphk_checkpoint_save(sphk_ctx* c, const char* path, const sphk_state_config* config, const sphk_state_section* sections,
                                    int n_sections) {
    if (!c || !path || !path[0] || !config || !valid_sections(sections, n_sections)) return SPHK_ERR_INVALID;
    std::vector<sphk_state_section> all(sections, sections + n_sections);
    ctx_sections(c, all);
    const int n = static_cast<int>(all.size());
    if (n > SPHK_STATE_MAX_SECTIONS) return SPHK_ERR_INVALID;
    if (int rc = stage_init(c)) return rc;
    StateStage* S = c->state;
    stage_join(S);                           // one save at a time: the pinned buffer is the previous save's until its write ends
    std::vector<Entry> table(static_cast<size_t>(n));
    unsigned long long payload = 0;
    for (int i = 0; i < n; ++i) {
        Entry& t = table[i];
        std::memset(&t, 0, sizeof(t));
        std::memcpy(t.name, all[i].name, SPHK_STATE_NAME);
        t.offset = payload; t.bytes = all[i].bytes; t.elem = all[i].elem_size; t.host = static_cast<unsigned int>(all[i].host);
        payload += align16(t.bytes);
    }
    if (int rc = stage_reserve(S, static_cast<size_t>(payload ? payload : 16), true)) return rc;
    // the device sections: one pack launch on the step stream, then the copy on the side stream
    int nd = 0;
    std::vector<int> devIndex;
    for (int i = 0; i < n; ++i) {
        if (all[i].host) continue;
        S->tableHost[nd++] = PackEntry{static_cast<const unsigned char*>(all[i].ptr), S->dev + table[i].offset, all[i].bytes, 0};
        devIndex.push_back(i);
    }
    if (nd) {
        if (int rc = enqueue_pack(c, S, nd)) return rc;
    }
    SPHK_CUDA_TRY(cudaEventRecord(S->packed, c->stream));
    SPHK_CUDA_TRY(cudaStreamWaitEvent(S->copy, S->packed, 0));
    if (payload) SPHK_CUDA_TRY(cudaMemcpyAsync(S->pinned, S->dev, static_cast<size_t>(payload), cudaMemcpyDeviceToHost, S->copy));
    if (nd) SPHK_CUDA_TRY(cudaMemcpyAsync(S->sumsHost, S->sums, 8ull * nd, cudaMemcpyDeviceToHost, S->copy));
    SPHK_CUDA_TRY(cudaEventRecord(S->copied, S->copy));
    // the host sections as they are now
    std::vector<std::vector<unsigned char>> hostData(static_cast<size_t>(n));
    for (int i = 0; i < n; ++i) {
        if (!all[i].host) continue;
        const unsigned char* p = static_cast<const unsigned char*>(all[i].ptr);
        hostData[i].assign(p, p + all[i].bytes);
        table[i].sum = checksum_host(p, all[i].bytes);
    }
    for (Entry& t : table) t.offset += header_bytes(n);
    const sphk_state_config cfg = *config;
    // the first failure of the saves since the last sphk_checkpoint_wait stays until a wait reports it
    if (!S->pending) { S->result = 0; S->message.clear(); }
    S->pending = true;
    int device = 0;
    SPHK_CUDA_TRY(cudaGetDevice(&device));
    S->writer = std::thread([S, cfg, table, hostData = std::move(hostData), devIndex, payload, device, p = std::string(path)]() mutable {
        auto fail = [S](int rc, const std::string& why) { if (S->result == 0) { S->result = rc; S->message = why; } };
        cudaSetDevice(device);          // the context's device, not device 0
        const cudaError_t e = cudaEventSynchronize(S->copied);
        if (e != cudaSuccess) { fail(static_cast<int>(e), std::string("device copy failed: ") + cudaGetErrorString(e)); return; }
        const size_t hb = header_bytes(static_cast<int>(table.size()));
        for (size_t k = 0; k < devIndex.size(); ++k) table[devIndex[k]].sum = S->sumsHost[k];
        for (size_t i = 0; i < table.size(); ++i) {
            if (!table[i].host) continue;
            unsigned char* dst = S->pinned + (table[i].offset - hb);
            std::memset(dst, 0, static_cast<size_t>(align16(table[i].bytes)));
            if (table[i].bytes) std::memcpy(dst, hostData[i].data(), static_cast<size_t>(table[i].bytes));
        }
        const std::vector<unsigned char> header = make_header(cfg, table, hb + payload);
        std::string why;
        const int rc = write_file(p, header, S->pinned, static_cast<size_t>(payload), why);
        if (rc) fail(rc, why);
    });
    return SPHK_OK;
}

extern "C" int sphk_checkpoint_wait(sphk_ctx* c, char* msg, int msg_len) {
    if (!c) return SPHK_ERR_INVALID;
    if (msg && msg_len > 0) msg[0] = 0;
    StateStage* S = c->state;
    if (!S || !S->pending) return SPHK_OK;
    stage_join(S);
    S->pending = false;
    if (S->result) say(msg, msg_len, "%s", S->message.c_str());
    return S->result;
}

extern "C" int sphk_checkpoint_release(sphk_ctx* c) {
    if (!c) return SPHK_ERR_INVALID;
    StateStage* S = c->state;
    if (!S) return SPHK_OK;
    stage_join(S);
    if (S->copy) cudaStreamSynchronize(S->copy);
    cudaFree(S->dev); cudaFree(S->table); cudaFree(S->sums);
    if (S->pinned) cudaFreeHost(S->pinned);
    if (S->tableHost) cudaFreeHost(S->tableHost);
    if (S->sumsHost) cudaFreeHost(S->sumsHost);
    if (S->copy) cudaStreamDestroy(S->copy);
    if (S->packed) cudaEventDestroy(S->packed);
    if (S->copied) cudaEventDestroy(S->copied);
    delete S;
    c->state = nullptr;
    return SPHK_OK;
}

// ---- loading --------------------------------------------------------------------------------------------------------------------
extern "C" int sphk_state_open(const char* path, sphk_state_file** out, char* msg, int msg_len) {
    if (!path || !out) return SPHK_ERR_INVALID;
    *out = nullptr;
    FILE* fp = std::fopen(path, "rb");
    if (!fp) { say(msg, msg_len, "cannot open %s: %s", path, std::strerror(errno)); return SPHK_ERR_INVALID; }
    sphk_state_file* f = new sphk_state_file();
    unsigned char buf[1 << 16];
    size_t got;
    while ((got = std::fread(buf, 1, sizeof(buf), fp)) > 0) f->bytes.insert(f->bytes.end(), buf, buf + got);
    const bool readErr = std::ferror(fp) != 0;
    std::fclose(fp);
    auto refuse = [&](const char* fmt, auto... a) { say(msg, msg_len, fmt, a...); delete f; return SPHK_ERR_INVALID; };
    if (readErr) return refuse("cannot read %s", path);
    const std::vector<unsigned char>& b = f->bytes;
    if (b.size() < kFixed) return refuse("header: truncated (%zu bytes, the fixed part is %zu)", b.size(), kFixed);
    if (std::memcmp(b.data(), kMagic, 8) != 0) return refuse("header: bad magic (not a checkpoint file)");
    unsigned int version = 0, n = 0;
    unsigned long long hb = 0, fileBytes = 0, cfgHash = 0;
    std::memcpy(&version, b.data() + 8, 4);
    std::memcpy(&n, b.data() + 12, 4);
    std::memcpy(&hb, b.data() + 16, 8);
    std::memcpy(&fileBytes, b.data() + 24, 8);
    std::memcpy(&cfgHash, b.data() + 32, 8);
    if (version != SPHK_STATE_VERSION) return refuse("header: version %u, this library reads version %d", version, SPHK_STATE_VERSION);
    if (n > SPHK_STATE_MAX_SECTIONS) return refuse("header: %u sections (at most %d)", n, SPHK_STATE_MAX_SECTIONS);
    if (b.size() < kFixed + kEntry * n + 4) return refuse("header: truncated (%zu bytes)", b.size());
    unsigned int crc = 0;
    std::memcpy(&crc, b.data() + kFixed + kEntry * n, 4);
    if (crc != crc32(b.data(), kFixed + kEntry * n)) return refuse("header: CRC-32 mismatch");
    if (hb != header_bytes(static_cast<int>(n))) return refuse("header: header size %llu, expected %zu", hb, header_bytes(static_cast<int>(n)));
    if (fileBytes != b.size()) return refuse("payload: the file has %zu bytes, its header says %llu (truncated?)", b.size(), fileBytes);
    std::memcpy(&f->config, b.data() + 40, sizeof(sphk_state_config));
    if (cfgHash != checksum_host(b.data() + 40, sizeof(sphk_state_config))) return refuse("header: config hash mismatch");
    f->table.resize(n);
    if (n) std::memcpy(f->table.data(), b.data() + kFixed, kEntry * n);
    for (const Entry& t : f->table) {
        if (std::memchr(t.name, 0, SPHK_STATE_NAME) == nullptr) return refuse("section table: an unterminated name");
        if (t.offset < hb || t.offset % 16 || t.bytes > fileBytes || t.offset > fileBytes - t.bytes)
            return refuse("section '%s': offset %llu + %llu bytes outside the file", t.name, t.offset, t.bytes);
    }
    *out = f;
    return SPHK_OK;
}

extern "C" void sphk_state_close(sphk_state_file* f) { delete f; }

extern "C" int sphk_state_section_bytes(const sphk_state_file* f, const char* name, unsigned long long* bytes) {
    if (!f || !name || !bytes) return SPHK_ERR_INVALID;
    for (const Entry& t : f->table)
        if (std::strncmp(t.name, name, SPHK_STATE_NAME) == 0) { *bytes = t.bytes; return SPHK_OK; }
    return SPHK_ERR_INVALID;
}

// names the first field of the config record that differs
static bool config_differs(const sphk_state_config& a, const sphk_state_config& e, char* msg, int len) {
#define SPHK_CFG_INT(f) if (std::memcmp(&a.f, &e.f, sizeof(a.f)) != 0) { say(msg, len, "config: %s differs (file %lld, system %lld)", #f, (long long)a.f, (long long)e.f); return true; }
#define SPHK_CFG_FLT(f) if (std::memcmp(&a.f, &e.f, sizeof(a.f)) != 0) { say(msg, len, "config: %s differs (file %.9g, system %.9g)", #f, (double)a.f, (double)e.f); return true; }
    if (std::memcmp(a.solver, e.solver, sizeof(a.solver)) != 0) {
        say(msg, len, "config: solver differs (file %.16s, system %.16s)", a.solver, e.solver);
        return true;
    }
    SPHK_CFG_INT(capacity_fluid) SPHK_CFG_INT(capacity_boundary) SPHK_CFG_INT(n_boundary) SPHK_CFG_INT(n_bodies)
    SPHK_CFG_INT(cell_size[0]) SPHK_CFG_INT(cell_size[1]) SPHK_CFG_INT(cell_size[2]) SPHK_CFG_INT(flags)
    SPHK_CFG_FLT(space_size[0]) SPHK_CFG_FLT(space_size[1]) SPHK_CFG_FLT(space_size[2]) SPHK_CFG_FLT(cell_length)
    SPHK_CFG_FLT(radius) SPHK_CFG_FLT(dt) SPHK_CFG_FLT(m0) SPHK_CFG_FLT(rho0) SPHK_CFG_FLT(rho_boundary) SPHK_CFG_FLT(stiff)
    SPHK_CFG_FLT(visc) SPHK_CFG_FLT(surface_tension) SPHK_CFG_FLT(air_pressure)
    SPHK_CFG_FLT(gravity[0]) SPHK_CFG_FLT(gravity[1]) SPHK_CFG_FLT(gravity[2])
    SPHK_CFG_FLT(solver_args[0]) SPHK_CFG_FLT(solver_args[1]) SPHK_CFG_FLT(solver_args[2]) SPHK_CFG_FLT(solver_args[3])
#undef SPHK_CFG_INT
#undef SPHK_CFG_FLT
    if (a.bodies_hash != e.bodies_hash) { say(msg, len, "config: bodies differ (points, masses or inertias)"); return true; }
    if (a.open_hash != e.open_hash) { say(msg, len, "config: emitters or sinks differ"); return true; }
    if (a.settings_hash != e.settings_hash) {
        say(msg, len, "config: settings differ (vorticity, viscosity, rheology, thermal, adhesion or adaptive rule)");
        return true;
    }
    return false;
}

extern "C" int sphk_checkpoint_load(sphk_ctx* c, const sphk_state_file* f, const sphk_state_config* expect,
                                    const sphk_state_section* sections, int n_sections, char* msg, int msg_len) {
    if (!c || !f || !expect || !valid_sections(sections, n_sections)) return SPHK_ERR_INVALID;
    if (msg && msg_len > 0) msg[0] = 0;
    if (config_differs(f->config, *expect, msg, msg_len)) return SPHK_ERR_INVALID;
    std::vector<sphk_state_section> all(sections, sections + n_sections);
    ctx_sections(c, all);
    if (all.size() != f->table.size()) {
        say(msg, msg_len, "section table: the file has %zu sections, the system %zu", f->table.size(), all.size());
        return SPHK_ERR_INVALID;
    }
    for (size_t i = 0; i < all.size(); ++i) {
        const Entry& t = f->table[i];
        if (std::strncmp(t.name, all[i].name, SPHK_STATE_NAME) != 0) {
            say(msg, msg_len, "section %zu: the file has '%s', the system expects '%s'", i, t.name, all[i].name);
            return SPHK_ERR_INVALID;
        }
        if (t.bytes != all[i].bytes || t.elem != all[i].elem_size || t.host != static_cast<unsigned int>(all[i].host)) {
            say(msg, msg_len, "section '%s': the file has %llu bytes (element %u), the system holds %llu (element %u)", t.name, t.bytes,
                t.elem, all[i].bytes, all[i].elem_size);
            return SPHK_ERR_INVALID;
        }
    }
    const unsigned char* base = f->bytes.data();
    for (size_t i = 0; i < all.size(); ++i) {
        const Entry& t = f->table[i];
        if (t.host && checksum_host(base + t.offset, t.bytes) != t.sum) {
            say(msg, msg_len, "section '%s': checksum mismatch", t.name);
            return SPHK_ERR_INVALID;
        }
    }
    // the device sections: upload into the staging buffer, checksums on the device, then -- only if all pass -- scatter
    if (int rc = stage_init(c)) return rc;
    StateStage* S = c->state;
    stage_join(S);                 // (a save's result stays for sphk_checkpoint_wait)
    unsigned long long payload = 0;
    std::vector<unsigned long long> at(all.size(), 0);
    for (size_t i = 0; i < all.size(); ++i)
        if (!all[i].host) { at[i] = payload; payload += align16(f->table[i].bytes); }
    if (int rc = stage_reserve(S, static_cast<size_t>(payload ? payload : 16), false)) return rc;
    int nd = 0;
    std::vector<size_t> devIndex;
    for (size_t i = 0; i < all.size(); ++i) {
        if (all[i].host) continue;
        const Entry& t = f->table[i];
        if (t.bytes) SPHK_CUDA_TRY(cudaMemcpyAsync(S->dev + at[i], base + t.offset, static_cast<size_t>(t.bytes), cudaMemcpyHostToDevice, c->stream));
        S->tableHost[nd++] = PackEntry{S->dev + at[i], nullptr, t.bytes, 0};
        devIndex.push_back(i);
    }
    if (nd) {
        if (int rc = enqueue_pack(c, S, nd)) return rc;
        SPHK_CUDA_TRY(cudaMemcpyAsync(S->sumsHost, S->sums, 8ull * nd, cudaMemcpyDeviceToHost, c->stream));
    }
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    for (int k = 0; k < nd; ++k) {
        const Entry& t = f->table[devIndex[k]];
        if (S->sumsHost[k] != t.sum) {
            say(msg, msg_len, "section '%s': checksum mismatch", t.name);
            return SPHK_ERR_INVALID;
        }
    }
    for (size_t i = 0; i < all.size(); ++i) {
        const Entry& t = f->table[i];
        if (!t.bytes) continue;
        if (all[i].host) std::memcpy(all[i].ptr, base + t.offset, static_cast<size_t>(t.bytes));
        else SPHK_CUDA_TRY(cudaMemcpyAsync(all[i].ptr, S->dev + at[i], static_cast<size_t>(t.bytes), cudaMemcpyDeviceToDevice, c->stream));
    }
    SPHK_CUDA_TRY(cudaStreamSynchronize(c->stream));
    return SPHK_OK;
}

extern "C" int sphk_checkpoint_invalidate(sphk_ctx* c) {
    if (!c) return SPHK_ERR_INVALID;
    // the fluid set must be searched again: no list, no permutation, no record scalar, positions dirty
    c->fluidSearched = false; c->permValid = false; c->countSettable = false;
    c->listEpoch = ~0ull; ++c->searchEpoch;
    c->posDirty = true; c->advected = true;
    c->sTag = nullptr;
    // DFSPH chunk activity and velocity epochs
    c->actMark = -1; c->tok = sphk_ctx::ErrTok{};
    c->velMark = -1; c->velArr = nullptr;
    const size_t chunks = static_cast<size_t>(c->capF) / 32 + 1;
    SPHK_CUDA_TRY(cudaMemsetAsync(c->chunkAct, 0, sizeof(unsigned int) * chunks, c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(c->chunkStamp, 0, sizeof(unsigned long long) * chunks, c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(c->chunkMark, 0, chunks, c->stream));
    // last-step statistics read as zero until the next step
    SPHK_CUDA_TRY(cudaMemsetAsync(c->loops, 0, 2 * sizeof(LoopState), c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(c->viscStats, 0, 2 * sizeof(float), c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(c->rheoStats, 0, 6 * sizeof(float), c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(c->heatStats, 0, 2 * sizeof(unsigned int), c->stream));
    SPHK_CUDA_TRY(cudaMemsetAsync(c->adhStats, 0, 2 * sizeof(unsigned int), c->stream));
    return SPHK_OK;
}
