// ob_api.cu -- C-ABI glue: error state, streams, staging of host buffers, LUT handles and the
// entry points declared in include/ouster_b200.h (everything except the decode path, which
// lives in ob_decode.cu).
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "ob_api_common.h"

namespace ob {

static thread_local std::string g_last_error;
static std::atomic<uint64_t> g_launches{0};

static std::atomic<uint64_t> g_family[OB_FAM_COUNT];
static const char* const kFamilies[OB_FAM_COUNT] = {"decode_pipe", "decode", "cloud", "normals", "voxel",
                                                    "voxel_map", "icp", "align", "zone"};

void count_launch(uint64_t n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
void count_launch_of(int family, uint64_t n) {
    if (family >= 0 && family < OB_FAM_COUNT) g_family[family].fetch_add(n, std::memory_order_relaxed);
}

ob_status fail(ob_status st, const std::string& msg) {
    g_last_error = msg;
    return st;
}
ob_status fail_cuda(cudaError_t e, const char* what) {
    g_last_error = std::string(what) + ": " + cudaGetErrorString(e);
    cudaGetLastError();  // clear sticky-less error state
    return OB_CUDA_ERROR;
}

static int env_int(const char* name, int dflt) {
    const char* v = std::getenv(name);
    return (v && *v) ? std::atoi(v) : dflt;
}

static std::mutex g_tun_mx;
static Tunables g_tun[64];
static char g_tun_have[64];

static Tunables& tunables_mut(int device) {
    if (device < 0 || device >= 64) device = 0;
    if (!g_tun_have[device]) {
        Tunables t;
        t.cloud_auto = (std::getenv("OB_CLOUD_TW") || std::getenv("OB_CLOUD_STAGES") || std::getenv("OB_CLOUD_CTAS_PER_SM") ||
                        std::getenv("OB_CLOUD_THREADS")) ? 0 : 1;
        t.cloud_tw = env_int("OB_CLOUD_TW", 512);
        t.cloud_stages = std::max(2, env_int("OB_CLOUD_STAGES", 3));
        t.cloud_threads = std::min(256, std::max(32, env_int("OB_CLOUD_THREADS", 128) / 32 * 32));  // compute threads
        t.cloud_ctas_per_sm = std::max(1, env_int("OB_CLOUD_CTAS_PER_SM", 3));
        t.cloud_pose_tw = std::max(16, env_int("OB_CLOUD_POSE_TW", 256));
        t.cloud_store_lag = env_int("OB_CLOUD_STORE_LAG", 1);
        t.cloud_pose_stages = std::max(2, env_int("OB_CLOUD_POSE_STAGES", 4));
        t.cloud_pose_ctas_per_sm = std::max(1, env_int("OB_CLOUD_POSE_CTAS_PER_SM", 5));
        t.cloud_pose_threads = std::min(256, std::max(32, env_int("OB_CLOUD_POSE_THREADS", 64) / 32 * 32));
        t.cloud_pose_rows = std::min(64, std::max(4, env_int("OB_CLOUD_POSE_ROWS", 16)));
        t.decode_stages = std::max(1, env_int("OB_DECODE_STAGES", 1));
        t.decode_threads = std::min(384, std::max(64, env_int("OB_DECODE_THREADS", 384) / 32 * 32));
        t.decode_ctas_per_sm = std::max(1, env_int("OB_DECODE_CTAS_PER_SM", 3));
        t.decode_tile_packets = std::max(0, env_int("OB_DECODE_TILE_PACKETS", 0));  // 0 = auto
        t.decode_prefetch = env_int("OB_DECODE_PREFETCH", 0);
        t.decode_runtime_plans = env_int("OB_DECODE_RUNTIME_PLANS", 0);
        t.decode_pipe = env_int("OB_DECODE_PIPE", 1);
        t.decode_pipe_warps = std::min(24, std::max(6, env_int("OB_DECODE_PIPE_WARPS", 24)));
        t.decode_pipe_dyn_rows = std::max(0, std::min(3, env_int("OB_DECODE_PIPE_DYN_ROWS", 3)));
        t.decode_pipe_tma_xyz = env_int("OB_DECODE_PIPE_TMA_XYZ", 0);  // measured: same time as the STG form (DESIGN.md, K2)
        t.decode_pipe_ctas = std::max(0, std::min(4, env_int("OB_DECODE_PIPE_CTAS", 0)));
        t.decode_pipe_helpers = std::max(0, std::min(6, env_int("OB_DECODE_PIPE_HELPERS", 0)));
        t.decode_pipe_lane_arrive = env_int("OB_DECODE_PIPE_LANE_ARRIVE", 1);
        t.decode_pipe_pk_split = std::min(16, std::max(1, env_int("OB_DECODE_PIPE_PK_SPLIT", 1)));
        t.decode_pipe_lut_split = std::min(8, std::max(1, env_int("OB_DECODE_PIPE_LUT_SPLIT", 1)));
        t.decode_pipe_prefetch = env_int("OB_DECODE_PIPE_PREFETCH", 0);  // measured: the extra L2 fills are evicted again (+19 % DRAM reads)
        t.force_generic = env_int("OB_FORCE_GENERIC", 0);
        int sm = 132;  // H100 SXM
        if (cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) {
            cudaGetLastError();
            sm = 132;
        }
        t.sm_count = sm > 0 ? sm : 132;
        g_tun[device] = t;
        g_tun_have[device] = 1;
    }
    return g_tun[device];
}

const Tunables& tunables(int device) {
    std::lock_guard<std::mutex> lk(g_tun_mx);
    return tunables_mut(device);
}

bool set_tunable(int device, const char* name, int value) {
    std::lock_guard<std::mutex> lk(g_tun_mx);
    Tunables& t = tunables_mut(device);
    const std::string n(name);
    if (n.rfind("cloud_", 0) == 0 && n != "cloud_store_lag" && n.find("pose") == std::string::npos) t.cloud_auto = 0;
    if (n == "cloud_tw") t.cloud_tw = std::max(4, value / 4 * 4);
    else if (n == "cloud_stages") t.cloud_stages = std::max(2, value);
    else if (n == "cloud_threads") t.cloud_threads = std::min(256, std::max(32, value / 32 * 32));
    else if (n == "cloud_ctas_per_sm") t.cloud_ctas_per_sm = std::max(1, value);
    else if (n == "cloud_pose_tw") t.cloud_pose_tw = std::max(16, value / 4 * 4);
    else if (n == "cloud_store_lag") t.cloud_store_lag = value ? 1 : 0;
    else if (n == "cloud_pose_stages") t.cloud_pose_stages = std::max(2, value);
    else if (n == "cloud_pose_ctas_per_sm") t.cloud_pose_ctas_per_sm = std::max(1, value);
    else if (n == "cloud_pose_threads") t.cloud_pose_threads = std::min(256, std::max(32, value / 32 * 32));
    else if (n == "cloud_pose_rows") t.cloud_pose_rows = std::min(64, std::max(4, value));
    else if (n == "decode_stages") t.decode_stages = std::max(1, value);
    else if (n == "decode_threads") t.decode_threads = std::min(384, std::max(64, value / 32 * 32));
    else if (n == "decode_ctas_per_sm") t.decode_ctas_per_sm = std::max(1, value);
    else if (n == "decode_tile_packets") t.decode_tile_packets = std::max(0, value);
    else if (n == "decode_prefetch") t.decode_prefetch = value;
    else if (n == "decode_runtime_plans") t.decode_runtime_plans = value ? 1 : 0;
    else if (n == "decode_pipe") t.decode_pipe = value ? 1 : 0;
    else if (n == "decode_pipe_warps") t.decode_pipe_warps = std::min(24, std::max(6, value));
    else if (n == "decode_pipe_prefetch") t.decode_pipe_prefetch = value;
    else if (n == "decode_pipe_tma_xyz") t.decode_pipe_tma_xyz = value ? 1 : 0;
    else if (n == "decode_pipe_ctas") t.decode_pipe_ctas = std::max(0, std::min(4, value));
    else if (n == "decode_pipe_helpers") t.decode_pipe_helpers = std::max(0, std::min(6, value));
    else if (n == "decode_pipe_lane_arrive") t.decode_pipe_lane_arrive = value ? 1 : 0;
    else if (n == "decode_pipe_pk_split") t.decode_pipe_pk_split = std::min(16, std::max(1, value));
    else if (n == "decode_pipe_lut_split") t.decode_pipe_lut_split = std::min(8, std::max(1, value));
    else if (n == "decode_pipe_dyn_rows") t.decode_pipe_dyn_rows = std::max(0, std::min(3, value));
    else if (n == "force_generic") t.force_generic = value;
    else return false;
    return true;
}

// ---------------------------------------------------------------------------------------------
// pointer classification and staging
// ---------------------------------------------------------------------------------------------
bool is_device_ptr(const void* p) {
    if (p == nullptr) return false;
    cudaPointerAttributes at;
    cudaError_t e = cudaPointerGetAttributes(&at, p);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

Staging::~Staging() {
    // scratch is released in stream order; host-visible results are final after ob_stream_sync
    for (void* p : scratch_) cudaFreeAsync(p, st_);
}

cudaError_t Staging::in(const void* p, size_t bytes, const void** dev) {
    if (bytes == 0 || p == nullptr) {
        *dev = p;
        return cudaSuccess;
    }
    if (is_device_ptr(p)) {
        *dev = p;
        return cudaSuccess;
    }
    void* d = nullptr;
    cudaError_t e = cudaMallocAsync(&d, bytes, st_);
    if (e != cudaSuccess) return e;
    scratch_.push_back(d);
    e = cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, st_);
    *dev = d;
    return e;
}

cudaError_t Staging::out(void* p, size_t bytes, void** dev) {
    if (bytes == 0 || p == nullptr) {
        *dev = p;
        return cudaSuccess;
    }
    if (is_device_ptr(p)) {
        *dev = p;
        return cudaSuccess;
    }
    void* d = nullptr;
    cudaError_t e = cudaMallocAsync(&d, bytes, st_);
    if (e != cudaSuccess) return e;
    scratch_.push_back(d);
    pending_.push_back({p, d, bytes});
    *dev = d;
    return cudaSuccess;
}

cudaError_t Staging::inout(void* p, size_t bytes, void** dev) {
    const void* d = nullptr;
    cudaError_t e = in(p, bytes, &d);
    if (e != cudaSuccess) return e;
    if (d != p) pending_.push_back({p, const_cast<void*>(d), bytes});
    *dev = const_cast<void*>(d);
    return cudaSuccess;
}

cudaError_t Staging::scratch(size_t bytes, void** dev) {
    void* d = nullptr;
    cudaError_t e = cudaMallocAsync(&d, bytes ? bytes : 16, st_);
    if (e != cudaSuccess) return e;
    scratch_.push_back(d);
    *dev = d;
    return cudaSuccess;
}

cudaError_t Staging::flush() {
    for (const Pending& q : pending_) {
        cudaError_t e = cudaMemcpyAsync(q.host, q.dev, q.bytes, cudaMemcpyDeviceToHost, st_);
        if (e != cudaSuccess) return e;
    }
    pending_.clear();
    return cudaSuccess;
}

ob_status require_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        cudaGetLastError();
        return fail(OB_NO_DEVICE,
                    "no CUDA device available: the ouster_b200 compute path has no CPU fallback");
    }
    if (device < 0 || device >= n) return fail(OB_INVALID_ARGUMENT, "invalid CUDA device index");
    e = cudaSetDevice(device);
    if (e != cudaSuccess) return fail_cuda(e, "cudaSetDevice");
    return OB_OK;
}

// reduce pixel_shift_by_row to rotation offsets in [0, w): d[u][j] = g[u][(j - off) mod w]
// (impl/lidar_frame_impl.h:756; true mathematical modulo -- identical to the reference's
// size_t expression for every power-of-two width, see DESIGN.md for other widths)
void reduce_shifts(const int32_t* shifts, size_t h, size_t w, int inverse, std::vector<uint16_t>& out) {
    out.resize(h);
    const long long W = static_cast<long long>(w);
    for (size_t u = 0; u < h; ++u) {
        long long s = inverse ? -static_cast<long long>(shifts[u]) : static_cast<long long>(shifts[u]);
        long long m = s % W;
        if (m < 0) m += W;
        out[u] = static_cast<uint16_t>(m);
    }
}

}  // namespace ob

using namespace ob;

struct ob_stream {
    int device;
    cudaStream_t st;
    bool owned;
    // small device-resident tables (frame tables of the decode / encode launches) kept across calls:
    // a steady-state caller passes the same pointers again and again, and re-uploading an identical
    // table costs a host-staged H2D copy per launch during which the GPU idles
    struct Table {
        void* dev{nullptr};
        size_t cap{0};
        std::vector<uint8_t> host;
    } tables[2];
};

struct ob_lut {
    int device;
    int dtype;
    size_t h, w;
    void* dir;
    void* off;
    // LUT-free mode (LUTs built from per-beam intrinsics only): device LutAnalyticT<T> + its tables
    void* an{nullptr};
    void* an_row{nullptr};
    void* an_col{nullptr};
    bool analytic_on{false};
};

// used by ob_decode.cu
namespace ob {
void lut_view(const ob_lut* lut, const void** dir, const void** off, int* dtype, size_t* h,
              size_t* w, int* device) {
    *dir = lut->dir;
    *off = lut->off;
    *dtype = lut->dtype;
    *h = lut->h;
    *w = lut->w;
    *device = lut->device;
}
const void* lut_analytic(const ob_lut* lut) { return lut->analytic_on ? lut->an : nullptr; }
cudaStream_t stream_handle(ob_stream* s) { return s->st; }

cudaError_t stream_table(ob_stream* s, int which, const void* host, size_t bytes, const void** dev) {
    ob_stream::Table& t = s->tables[which & 1];
    if (t.dev != nullptr && t.host.size() == bytes && std::memcmp(t.host.data(), host, bytes) == 0) {
        *dev = t.dev;  // identical to what the device already holds
        return cudaSuccess;
    }
    if (bytes > t.cap) {
        if (t.dev) {
            cudaError_t e = cudaStreamSynchronize(s->st);  // a running launch may still read the old table
            if (e != cudaSuccess) return e;
            cudaFree(t.dev);
            t.dev = nullptr;
            t.cap = 0;
        }
        const size_t cap = std::max<size_t>(bytes * 2, 4096);
        cudaError_t e = cudaMalloc(&t.dev, cap);
        if (e != cudaSuccess) return e;
        t.cap = cap;
    }
    t.host.assign(static_cast<const uint8_t*>(host), static_cast<const uint8_t*>(host) + bytes);
    // stream-ordered: lands after every earlier launch of this stream that reads the previous contents
    cudaError_t e = cudaMemcpyAsync(t.dev, t.host.data(), bytes, cudaMemcpyHostToDevice, s->st);
    if (e != cudaSuccess) {
        t.host.clear();
        return e;
    }
    *dev = t.dev;
    return cudaSuccess;
}
int stream_device(ob_stream* s) { return s->device; }
}  // namespace ob

extern "C" {

int ob_abi_version(void) { return OB_ABI_VERSION; }

size_t ob_abi_sizeof(const char* name) {
    if (!name) return 0;
    const std::string n(name);
    if (n == "ob_cloud_io") return sizeof(ob_cloud_io);
    if (n == "ob_field_desc") return sizeof(ob_field_desc);
    if (n == "ob_packet_layout") return sizeof(ob_packet_layout);
    if (n == "ob_decode_io") return sizeof(ob_decode_io);
    if (n == "ob_decode_batch") return sizeof(ob_decode_batch);
    if (n == "ob_dewarp_frame_io") return sizeof(ob_dewarp_frame_io);
    if (n == "ob_normals_io") return sizeof(ob_normals_io);
    if (n == "ob_encode_io") return sizeof(ob_encode_io);
    if (n == "ob_dewarp_frames_io") return sizeof(ob_dewarp_frames_io);
    if (n == "ob_voxel_io") return sizeof(ob_voxel_io);
    if (n == "ob_point_rows") return sizeof(ob_point_rows);
    if (n == "ob_voxel_map_cull_io") return sizeof(ob_voxel_map_cull_io);
    if (n == "ob_voxel_query_io") return sizeof(ob_voxel_query_io);
    if (n == "ob_icp_io") return sizeof(ob_icp_io);
    if (n == "ob_icp_system_io") return sizeof(ob_icp_system_io);
    if (n == "ob_cloud_align_io") return sizeof(ob_cloud_align_io);
    if (n == "ob_cloud_nearest_io") return sizeof(ob_cloud_nearest_io);
    if (n == "ob_zone_desc") return sizeof(ob_zone_desc);
    if (n == "ob_zone_render_io") return sizeof(ob_zone_render_io);
    if (n == "ob_zone_live") return sizeof(ob_zone_live);
    if (n == "ob_zone_state") return sizeof(ob_zone_state);
    return 0;
}

const char* ob_last_error(void) { return g_last_error.c_str(); }

int ob_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
}

uint64_t ob_kernel_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

uint64_t ob_kernel_launch_count_of(const char* name) {
    if (!name) return 0;
    for (int i = 0; i < OB_FAM_COUNT; ++i)
        if (std::string(name) == kFamilies[i]) return g_family[i].load(std::memory_order_relaxed);
    return 0;
}

ob_status ob_set_tunable(int device, const char* name, int value) {
    if (!name || !set_tunable(device, name, value)) return fail(OB_INVALID_ARGUMENT, "unknown tunable");
    return OB_OK;
}

ob_status ob_stream_create(int device, ob_stream** out) {
    if (!out) return fail(OB_INVALID_ARGUMENT, "null output pointer");
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st;
    cudaError_t e = cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking);
    if (e != cudaSuccess) return fail_cuda(e, "cudaStreamCreate");
    // keep the stream-ordered pool from trimming between calls
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t thr = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    ob_stream* ns = new ob_stream;
    ns->device = device;
    ns->st = st;
    ns->owned = true;
    *out = ns;
    return OB_OK;
}

ob_status ob_stream_wrap(int device, void* cuda_stream, ob_stream** out) {
    if (!out) return fail(OB_INVALID_ARGUMENT, "null output pointer");
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t thr = ~0ull;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    ob_stream* ns = new ob_stream;
    ns->device = device;
    ns->st = static_cast<cudaStream_t>(cuda_stream);
    ns->owned = false;
    *out = ns;
    return OB_OK;
}

ob_status ob_stream_sync(ob_stream* s) {
    if (!s) return fail(OB_INVALID_ARGUMENT, "null stream");
    cudaError_t e = cudaStreamSynchronize(s->st);
    if (e != cudaSuccess) return fail_cuda(e, "cudaStreamSynchronize");
    return OB_OK;
}

void* ob_stream_cuda_handle(ob_stream* s) { return s ? static_cast<void*>(s->st) : nullptr; }

ob_status ob_stream_destroy(ob_stream* s) {
    if (!s) return OB_OK;
    bool have_tables = false;
    for (auto& t : s->tables) have_tables |= t.dev != nullptr;
    if (s->owned || have_tables) cudaStreamSynchronize(s->st);
    for (auto& t : s->tables)
        if (t.dev) cudaFree(t.dev);
    if (s->owned) cudaStreamDestroy(s->st);
    delete s;
    return OB_OK;
}

ob_status ob_host_alloc(size_t bytes, void** out) {
    if (!out) return fail(OB_INVALID_ARGUMENT, "null output pointer");
    if (ob_device_count() <= 0) return fail(OB_NO_DEVICE, "no CUDA device available");
    cudaError_t e = cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault);
    if (e != cudaSuccess) return fail_cuda(e, "cudaHostAlloc");
    return OB_OK;
}

ob_status ob_host_free(void* p) {
    if (!p) return OB_OK;
    cudaError_t e = cudaFreeHost(p);
    if (e != cudaSuccess) return fail_cuda(e, "cudaFreeHost");
    return OB_OK;
}

// ---------------------------------------------------------------------------------------------
// LUT
// ---------------------------------------------------------------------------------------------
static size_t dtype_size(int dtype) { return dtype == OB_F64 ? 8 : 4; }

}  // extern "C"

// Per-row / per-column tables of the LUT-free projection, from the same intrinsics and in the same
// double arithmetic as make_xyz_lut (ouster_core/src/xyzlut.cpp:24-86), then cast to the LUT's scalar.
template <typename T>
static cudaError_t build_analytic(ob_lut* l, double range_unit, const double* b2l, const double* tr,
                                  const double* az_deg, const double* alt_deg) {
    const size_t h = l->h, w = l->w;
    std::vector<T> row(h * 4), col(w * 2);
    const double b03 = b2l[3], b23 = b2l[11];
    double dist = b03;
    if (b23 != 0) dist = std::sqrt(b03 * b03 + b23 * b23);
    for (size_t r = 0; r < h; ++r) {
        const double az = -az_deg[r] * M_PI / 180.0, alt = alt_deg[r] * M_PI / 180.0;
        row[4 * r + 0] = static_cast<T>(std::cos(az) * std::cos(alt));
        row[4 * r + 1] = static_cast<T>(std::sin(az) * std::cos(alt));
        row[4 * r + 2] = static_cast<T>(std::sin(alt));
        row[4 * r + 3] = 0;
    }
    const double azimuth_radians = M_PI * 2.0 / static_cast<double>(w);
    for (size_t c = 0; c < w; ++c) {
        const double enc = 2.0 * M_PI - static_cast<double>(c) * azimuth_radians;
        col[2 * c + 0] = static_cast<T>(std::cos(enc));
        col[2 * c + 1] = static_cast<T>(std::sin(enc));
    }
    LutAnalyticT<T> a;
    a.dist = static_cast<T>(dist);
    a.b03 = static_cast<T>(b03);
    a.b23 = static_cast<T>(b23);
    for (int j = 0; j < 3; ++j)
        for (int k = 0; k < 4; ++k) a.m[4 * j + k] = static_cast<T>(tr[4 * j + k] * range_unit);
    cudaError_t e = cudaMalloc(&l->an_row, row.size() * sizeof(T));
    if (e == cudaSuccess) e = cudaMalloc(&l->an_col, col.size() * sizeof(T));
    if (e == cudaSuccess) e = cudaMalloc(&l->an, sizeof(a));
    if (e == cudaSuccess) e = cudaMemcpy(l->an_row, row.data(), row.size() * sizeof(T), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(l->an_col, col.data(), col.size() * sizeof(T), cudaMemcpyHostToDevice);
    a.row = static_cast<const T*>(l->an_row);
    a.col = static_cast<const T*>(l->an_col);
    if (e == cudaSuccess) e = cudaMemcpy(l->an, &a, sizeof(a), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) {
        cudaFree(l->an);
        cudaFree(l->an_row);
        cudaFree(l->an_col);
        l->an = l->an_row = l->an_col = nullptr;
    }
    return e;
}

extern "C" {

ob_status ob_lut_create(ob_dtype dtype, const void* direction, const void* offset, size_t h,
                        size_t w, int device, ob_lut** out) {
    if (!out || !direction || !offset) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (dtype != OB_F32 && dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "unknown dtype");
    if (w == 0 || h == 0)
        return fail(OB_INVALID_ARGUMENT, "lut dimensions must be greater than zero");
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    const size_t bytes = h * w * 3 * dtype_size(dtype);
    void *d = nullptr, *o = nullptr;
    cudaError_t e = cudaMalloc(&d, bytes);
    if (e != cudaSuccess) return fail_cuda(e, "cudaMalloc(lut)");
    e = cudaMalloc(&o, bytes);
    if (e != cudaSuccess) {
        cudaFree(d);
        return fail_cuda(e, "cudaMalloc(lut)");
    }
    e = cudaMemcpy(d, direction, bytes, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(o, offset, bytes, cudaMemcpyDefault);
    if (e != cudaSuccess) {
        cudaFree(d);
        cudaFree(o);
        return fail_cuda(e, "cudaMemcpy(lut)");
    }
    *out = new ob_lut{device, static_cast<int>(dtype), h, w, d, o};
    return OB_OK;
}

ob_status ob_lut_from_intrinsics(ob_dtype dtype, size_t w, size_t h, double range_unit,
                                 const double* b2l, const double* transform, const double* az,
                                 size_t n_az, const double* alt, size_t n_alt, int device,
                                 ob_lut** out) {
    if (!out) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (dtype != OB_F32 && dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "unknown dtype");
    // validation order and texts of make_xyz_lut, ouster_core/src/xyzlut.cpp:14-21
    if (w == 0 || h == 0)
        return fail(OB_INVALID_ARGUMENT, "lut dimensions must be greater than zero");
    if ((n_az != h || n_alt != h) && (n_az != w * h || n_alt != w * h))
        return fail(OB_INVALID_ARGUMENT, "unexpected frame dimensions");
    if (!b2l || !transform || !az || !alt) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;

    const size_t n3 = w * h * 3;
    double *daz = nullptr, *dalt = nullptr, *dd = nullptr, *doff = nullptr;
    cudaError_t e = cudaMalloc(&daz, n_az * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dalt, n_alt * 8);
    if (e == cudaSuccess) e = cudaMalloc(&dd, n3 * 8);
    if (e == cudaSuccess) e = cudaMalloc(&doff, n3 * 8);
    if (e == cudaSuccess) e = cudaMemcpy(daz, az, n_az * 8, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(dalt, alt, n_alt * 8, cudaMemcpyDefault);
    if (e == cudaSuccess)
        e = launch_make_lut(w, h, range_unit, b2l, transform, daz, n_az, dalt, n_alt, dd, doff, 0);
    void *rd = dd, *ro = doff;
    if (e == cudaSuccess && dtype == OB_F32) {
        float *fd = nullptr, *fo = nullptr;
        e = cudaMalloc(&fd, n3 * 4);
        if (e == cudaSuccess) e = cudaMalloc(&fo, n3 * 4);
        if (e == cudaSuccess) e = launch_cast_f64_f32(dd, fd, n3, 0);
        if (e == cudaSuccess) e = launch_cast_f64_f32(doff, fo, n3, 0);
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
        if (e == cudaSuccess) {
            cudaFree(dd);
            cudaFree(doff);
            dd = doff = nullptr;
            rd = fd;
            ro = fo;
        } else {
            cudaFree(fd);
            cudaFree(fo);
        }
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    cudaFree(daz);
    cudaFree(dalt);
    if (e != cudaSuccess) {
        cudaFree(dd);
        cudaFree(doff);
        return fail_cuda(e, "ob_lut_from_intrinsics");
    }
    ob_lut* l = new ob_lut{device, static_cast<int>(dtype), h, w, rd, ro};
    if (n_az == h && n_alt == h) {  // per-beam angles: the LUT-free tables exist (off until ob_lut_set_analytic)
        cudaError_t ea = dtype == OB_F64 ? build_analytic<double>(l, range_unit, b2l, transform, az, alt)
                                         : build_analytic<float>(l, range_unit, b2l, transform, az, alt);
        if (ea != cudaSuccess) cudaGetLastError();  // optional feature: the LUT itself is complete
    }
    *out = l;
    return OB_OK;
}

ob_status ob_lut_set_analytic(ob_lut* lut, int enable) {
    if (!lut) return fail(OB_INVALID_ARGUMENT, "null lut");
    if (enable && !lut->an)
        return fail(OB_INVALID_ARGUMENT, "LUT-free projection needs a lut built from per-beam intrinsics");
    lut->analytic_on = enable != 0;
    return OB_OK;
}

int ob_lut_is_analytic(const ob_lut* lut) { return lut && lut->analytic_on ? 1 : 0; }

ob_status ob_lut_download(const ob_lut* lut, void* direction, void* offset) {
    if (!lut || !direction || !offset) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const size_t bytes = lut->h * lut->w * 3 * dtype_size(lut->dtype);
    cudaSetDevice(lut->device);
    cudaError_t e = cudaMemcpy(direction, lut->dir, bytes, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(offset, lut->off, bytes, cudaMemcpyDefault);
    if (e != cudaSuccess) return fail_cuda(e, "ob_lut_download");
    return OB_OK;
}

ob_status ob_lut_info(const ob_lut* lut, size_t* h, size_t* w, int* dtype, int* device) {
    if (!lut) return fail(OB_INVALID_ARGUMENT, "null lut");
    if (h) *h = lut->h;
    if (w) *w = lut->w;
    if (dtype) *dtype = lut->dtype;
    if (device) *device = lut->device;
    return OB_OK;
}

ob_status ob_lut_device_ptrs(const ob_lut* lut, void** direction, void** offset) {
    if (!lut) return fail(OB_INVALID_ARGUMENT, "null lut");
    if (direction) *direction = lut->dir;
    if (offset) *offset = lut->off;
    return OB_OK;
}

ob_status ob_lut_destroy(ob_lut* lut) {
    if (!lut) return OB_OK;
    cudaSetDevice(lut->device);
    forget_lut_tensor_maps(lut->dir);
    cudaFree(lut->dir);
    cudaFree(lut->off);
    cudaFree(lut->an);
    cudaFree(lut->an_row);
    cudaFree(lut->an_col);
    delete lut;
    return OB_OK;
}


// ---------------------------------------------------------------------------------------------
// scan -> cloud
// ---------------------------------------------------------------------------------------------
}  // extern "C"

template <typename T>
static ob_status scan_to_cloud_t(const ob_lut* lut, const uint16_t* shift, const ob_cloud_io* io,
                                 ob_stream* s) {
    const size_t n_px = lut->h * lut->w;
    const uint32_t F = io->n_frames, R = io->n_returns;
    Staging stg(s->st);
    // extent (in elements) spanned by a strided [F][R][n] array
    auto extent = [&](size_t fs, size_t rs, size_t n) {
        return (F - 1) * fs + (R - 1) * rs + n;
    };
    CloudArgs<T> a;
    a.dir = static_cast<const T*>(lut->dir);
    a.off = static_cast<const T*>(lut->off);
    a.analytic = lut->analytic_on ? static_cast<const LutAnalyticT<T>*>(lut->an) : nullptr;
    a.range_fs = io->range_frame_stride;
    a.range_rs = io->range_return_stride;
    a.xyz_fs = io->xyz_frame_stride;
    a.xyz_rs = io->xyz_return_stride;
    a.rd_fs = io->rd_frame_stride;
    a.rd_rs = io->rd_return_stride;
    a.xd_fs = io->xd_frame_stride;
    a.xd_rs = io->xd_return_stride;
    a.H = static_cast<int>(lut->h);
    a.W = static_cast<int>(lut->w);
    a.n_returns = static_cast<int>(R);
    a.n_frames = F;
    a.shift = shift;
    const void* din = nullptr;
    void* dout = nullptr;
    cudaError_t e = stg.in(io->range, extent(a.range_fs, a.range_rs, n_px) * 4, &din);
    if (e != cudaSuccess) return fail_cuda(e, "stage range");
    a.range = static_cast<const uint32_t*>(din);
    a.xyz = nullptr;
    a.rd = nullptr;
    a.xd = nullptr;
    if (io->xyz) {
        e = stg.out(io->xyz, extent(a.xyz_fs, a.xyz_rs, n_px * 3) * sizeof(T), &dout);
        if (e != cudaSuccess) return fail_cuda(e, "stage xyz");
        a.xyz = static_cast<T*>(dout);
    }
    if (io->range_destaggered) {
        e = stg.out(io->range_destaggered, extent(a.rd_fs, a.rd_rs, n_px) * 4, &dout);
        if (e != cudaSuccess) return fail_cuda(e, "stage range_destaggered");
        a.rd = static_cast<uint32_t*>(dout);
    }
    if (io->xyz_destaggered) {
        e = stg.out(io->xyz_destaggered, extent(a.xd_fs, a.xd_rs, n_px * 3) * sizeof(T), &dout);
        if (e != cudaSuccess) return fail_cuda(e, "stage xyz_destaggered");
        a.xd = static_cast<T*>(dout);
    }
    if (io->poses) {
        const size_t pn = static_cast<size_t>(lut->w) * 16;
        e = stg.in(io->poses, ((F - 1) * io->poses_frame_stride + pn) * sizeof(T), &din);
        if (e != cudaSuccess) return fail_cuda(e, "stage poses");
        a.poses = static_cast<const T*>(din);
        a.poses_fs = io->poses_frame_stride;
    }
    e = launch_cloud<T>(a, s->device, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "scan_to_cloud launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "scan_to_cloud D2H");
    return OB_OK;
}

extern "C" {

ob_status ob_scan_to_cloud(const ob_lut* lut, const int32_t* shifts, size_t n_shifts,
                           const ob_cloud_io* io, ob_stream* s) {
    if (!lut || !io || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (!io->range) return fail(OB_INVALID_ARGUMENT, "null range image");
    if (io->n_returns < 1 || io->n_returns > OB_MAX_RETURNS)
        return fail(OB_INVALID_ARGUMENT, "n_returns must be 1 or 2");
    if (io->n_frames == 0) return OB_OK;
    const bool needs_shift = io->range_destaggered || io->xyz_destaggered;
    if (needs_shift) {
        if (!shifts || n_shifts != lut->h)
            return fail(OB_INVALID_ARGUMENT, "image height does not match shifts size");
        if (lut->h > static_cast<size_t>(kMaxRows))
            return fail(OB_INVALID_ARGUMENT, "fused destagger supports at most 512 rows");
    }
    if (lut->w > 65535) return fail(OB_INVALID_ARGUMENT, "frame width exceeds 65535 columns");
    if (io->poses && !io->xyz && !io->xyz_destaggered)
        return fail(OB_INVALID_ARGUMENT, "poses given without an xyz output");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    if (lut->device != s->device) return fail(OB_INVALID_ARGUMENT, "lut and stream are on different devices");
    std::vector<uint16_t> sh;
    if (needs_shift) reduce_shifts(shifts, lut->h, lut->w, 0, sh);
    if (lut->dtype == OB_F64) return scan_to_cloud_t<double>(lut, needs_shift ? sh.data() : nullptr, io, s);
    return scan_to_cloud_t<float>(lut, needs_shift ? sh.data() : nullptr, io, s);
}

ob_status ob_cartesian(const ob_lut* lut, const uint32_t* range, size_t n_pixels, void* xyz,
                       ob_stream* s) {
    if (!lut || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (n_pixels != lut->h * lut->w) return fail(OB_INVALID_ARGUMENT, "unexpected image dimensions");
    if (!range || !xyz) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_cloud_io io;
    std::memset(&io, 0, sizeof(io));
    io.n_frames = 1;
    io.n_returns = 1;
    io.range = range;
    io.xyz = xyz;
    return ob_scan_to_cloud(lut, nullptr, 0, &io, s);
}

ob_status ob_dewarp(ob_dtype dtype, const void* points, const void* poses, size_t n_points,
                    size_t n_poses, void* out, ob_stream* s) {
    if (!s) return fail(OB_INVALID_ARGUMENT, "null stream");
    if (dtype != OB_F32 && dtype != OB_F64) return fail(OB_INVALID_ARGUMENT, "unknown dtype");
    if (n_points == 0) return OB_OK;
    if (!points || !poses || !out) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (n_poses == 0 || n_points % n_poses != 0)
        return fail(OB_RUNTIME_ERROR, "Number of points per set must match number of poses");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    const size_t esz = dtype == OB_F64 ? 8 : 4;
    Staging stg(s->st);
    const void *dp = nullptr, *dq = nullptr;
    void* dout = nullptr;
    cudaError_t e = stg.in(points, n_points * 3 * esz, &dp);
    if (e == cudaSuccess) e = stg.in(poses, n_poses * 16 * esz, &dq);
    if (e == cudaSuccess) e = stg.out(out, n_points * 3 * esz, &dout);
    if (e != cudaSuccess) return fail_cuda(e, "stage dewarp buffers");
    const size_t H = n_points / n_poses;
    if (dtype == OB_F64)
        e = launch_dewarp<double>(static_cast<const double*>(dp), static_cast<const double*>(dq),
                                  static_cast<double*>(dout), H, n_poses, s->st);
    else
        e = launch_dewarp<float>(static_cast<const float*>(dp), static_cast<const float*>(dq),
                                 static_cast<float*>(dout), H, n_poses, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "dewarp launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "dewarp D2H");
    return OB_OK;
}

// Shared driver of ob_dewarp_frame / ob_dewarp_frames: frame table upload, ONE kernel launch, then the
// device-side counts.  Results for device outputs are complete in stream order; the only host wait is the
// one a host-memory result needs anyway.
static ob_status run_dewarp(std::vector<K3Frame>& hf, int dtype, uint32_t min_r, uint32_t max_r, void* points,
                            size_t capacity, uint32_t* frame_idx, uint32_t* col_idx, uint64_t* timestamps_out,
                            size_t* counts, size_t* n_points, Staging& stg, ob_stream* s) {
    unsigned n_blocks = 0, max_slabs = 0;
    for (K3Frame& f : hf) {
        f.first_block = n_blocks;
        n_blocks += f.n_cg;
        max_slabs = std::max(max_slabs, f.n_slabs);
    }
    const size_t esz = dtype_size(dtype);
    void *fdev = nullptr, *scan = nullptr, *o = nullptr;
    cudaError_t e = stg.scratch(hf.size() * sizeof(K3Frame), &fdev);
    if (e == cudaSuccess) e = stg.scratch(dewarp_scan_scratch_bytes(n_blocks, static_cast<unsigned>(hf.size())), &scan);
    if (e == cudaSuccess) e = cudaMemcpyAsync(fdev, hf.data(), hf.size() * sizeof(K3Frame), cudaMemcpyHostToDevice, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "frame table upload");
    // outputs: device pointers in place, host pointers through device scratch of `capacity` points
    const bool host_out = !is_device_ptr(points);
    void* dpts = points;
    uint32_t *dfi = frame_idx, *dci = col_idx;
    uint64_t* dts = timestamps_out;
    if (host_out) {
        e = stg.scratch(std::max<size_t>(1, capacity) * 3 * esz, &o);
        dpts = o;
        if (e == cudaSuccess && frame_idx) {
            e = stg.scratch(std::max<size_t>(1, capacity) * 4, &o);
            dfi = static_cast<uint32_t*>(o);
        }
        if (e == cudaSuccess && col_idx) {
            e = stg.scratch(std::max<size_t>(1, capacity) * 4, &o);
            dci = static_cast<uint32_t*>(o);
        }
        if (e == cudaSuccess && timestamps_out) {
            e = stg.scratch(std::max<size_t>(1, capacity) * 8, &o);
            dts = static_cast<uint64_t*>(o);
        }
        if (e != cudaSuccess) return fail_cuda(e, "stage dewarp outputs");
    }
    const unsigned long long* fend = nullptr;
    e = launch_dewarp_fused(static_cast<const K3Frame*>(fdev), static_cast<unsigned>(hf.size()), n_blocks, max_slabs,
                            min_r, max_r, dtype, scan, dpts, dfi, dci, dts, capacity, &fend, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "dewarp launch");
    if (is_device_ptr(n_points)) {
        // fully asynchronous form: the count stays on the device next to the points (a count above
        // `capacity` means the list was cut at `capacity` points; no error can be raised from here)
        if (host_out || counts) return fail(OB_INVALID_ARGUMENT, "a device-side count needs device outputs and no per-frame counts");
        e = cudaMemcpyAsync(n_points, fend + (hf.size() - 1), 8, cudaMemcpyDeviceToDevice, s->st);
        if (e != cudaSuccess) return fail_cuda(e, "dewarp count");
        return OB_OK;
    }
    std::vector<unsigned long long> ends(hf.size());
    e = cudaMemcpyAsync(ends.data(), fend, hf.size() * 8, cudaMemcpyDeviceToHost, s->st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s->st);
    if (e != cudaSuccess) return fail_cuda(e, "dewarp count");
    const unsigned long long total = ends.back();
    if (counts)
        for (size_t k = 0; k < hf.size(); ++k) counts[hf[k].index] = static_cast<size_t>(ends[k] - (k ? ends[k - 1] : 0ull));
    if (total > capacity) return fail(OB_INVALID_ARGUMENT, "output capacity too small");
    if (host_out && total) {
        e = cudaMemcpyAsync(points, dpts, total * 3 * esz, cudaMemcpyDeviceToHost, s->st);
        if (e == cudaSuccess && frame_idx) e = cudaMemcpyAsync(frame_idx, dfi, total * 4, cudaMemcpyDeviceToHost, s->st);
        if (e == cudaSuccess && col_idx) e = cudaMemcpyAsync(col_idx, dci, total * 4, cudaMemcpyDeviceToHost, s->st);
        if (e == cudaSuccess && timestamps_out)
            e = cudaMemcpyAsync(timestamps_out, dts, total * 8, cudaMemcpyDeviceToHost, s->st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(s->st);
        if (e != cudaSuccess) return fail_cuda(e, "dewarp D2H");
    }
    *n_points = static_cast<size_t>(total);
    return OB_OK;
}

static ob_status stage_k3_frame(const ob_lut* lut, const uint32_t* range, const double* poses, const uint32_t* status,
                                const uint64_t* timestamps, bool want_ts, unsigned index, Staging& stg, K3Frame* out) {
    K3Frame f{};
    f.H = static_cast<unsigned>(lut->h);
    f.W = static_cast<unsigned>(lut->w);
    f.n_cg = (f.W + 31) / 32;
    f.n_slabs = (f.H + 15) / 16;
    f.index = index;
    f.dir = lut->dir;
    f.off = lut->off;
    const size_t n_px = lut->h * lut->w;
    const void* d = nullptr;
    cudaError_t e = stg.in(range, n_px * 4, &d);
    f.range = static_cast<const uint32_t*>(d);
    if (e == cudaSuccess) e = stg.in(poses, lut->w * 16 * sizeof(double), &d);
    f.poses = static_cast<const double*>(d);
    if (e == cudaSuccess) e = stg.in(status, lut->w * 4, &d);
    f.status = static_cast<const uint32_t*>(d);
    if (e == cudaSuccess && want_ts) {
        e = stg.in(timestamps, lut->w * 8, &d);
        f.timestamps = static_cast<const uint64_t*>(d);
    }
    if (e != cudaSuccess) return fail_cuda(e, "stage dewarp inputs");
    *out = f;
    return OB_OK;
}

// same conversions as the reference (dewarp_impl.h:34-35); NaN / negative limits select nothing
static bool range_window(double min_range, double max_range, uint32_t* min_r, uint32_t* max_r) {
    const double lo = std::ceil(min_range * 1e3), hi = std::floor(max_range * 1e3);
    if (!(lo <= 4294967295.0) || !(hi >= 0.0) || !(lo <= hi)) return false;
    *min_r = lo <= 0.0 ? 0u : static_cast<uint32_t>(lo);
    *max_r = hi >= 4294967295.0 ? 0xffffffffu : static_cast<uint32_t>(hi);
    return true;
}

static ob_status zero_count(size_t* n_points, ob_stream* s) {
    if (is_device_ptr(n_points)) {
        cudaError_t e = cudaMemsetAsync(n_points, 0, 8, s->st);
        return e == cudaSuccess ? OB_OK : fail_cuda(e, "dewarp count");
    }
    *n_points = 0;
    return OB_OK;
}

ob_status ob_dewarp_frame(const ob_lut* lut, const ob_dewarp_frame_io* io, size_t* n_points, ob_stream* s) {
    if (!lut || !io || !n_points || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    rs = zero_count(n_points, s);
    if (rs != OB_OK) return rs;
    if (!io->range || !io->poses || !io->status || !io->points)
        return fail(OB_INVALID_ARGUMENT, "null range / poses / status / points");
    if (io->timestamps_out && !io->timestamps)
        return fail(OB_INVALID_ARGUMENT, "timestamps_out requested without column timestamps");
    if (lut->device != s->device) return fail(OB_INVALID_ARGUMENT, "lut and stream are on different devices");
    uint32_t min_r, max_r;
    if (!range_window(io->min_range, io->max_range, &min_r, &max_r)) return OB_OK;
    if (lut->h == 0 || lut->w == 0) return OB_OK;
    Staging stg(s->st);
    std::vector<K3Frame> hf(1);
    rs = stage_k3_frame(lut, io->range, io->poses, io->status, io->timestamps, io->timestamps_out != nullptr, 0, stg, &hf[0]);
    if (rs != OB_OK) return rs;
    return run_dewarp(hf, lut->dtype, min_r, max_r, io->points, io->capacity, nullptr, io->col_idx, io->timestamps_out,
                      nullptr, n_points, stg, s);
}

ob_status ob_dewarp_frames(const ob_dewarp_frames_io* frames, size_t n_frames, double min_range, double max_range,
                           void* points, size_t capacity, uint32_t* frame_idx, uint32_t* col_idx,
                           uint64_t* timestamps_out, size_t* counts, size_t* n_points, ob_stream* s) {
    if (!s || !n_points || (n_frames && !frames)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    rs = zero_count(n_points, s);
    if (rs != OB_OK) return rs;
    if (counts) std::fill(counts, counts + n_frames, static_cast<size_t>(0));
    if (n_frames == 0) return OB_OK;
    if (!points) return fail(OB_INVALID_ARGUMENT, "null points buffer");
    uint32_t min_r, max_r;
    if (!range_window(min_range, max_range, &min_r, &max_r)) return OB_OK;
    int dtype = -1;
    Staging stg(s->st);
    std::vector<K3Frame> hf;
    hf.reserve(n_frames);
    for (size_t i = 0; i < n_frames; ++i) {
        const ob_dewarp_frames_io& io = frames[i];
        if (!io.lut) continue;  // FrameSet::valid_indices(): empty slots of the set are skipped
        if (!io.range || !io.poses || !io.status) return fail(OB_INVALID_ARGUMENT, "null range / poses / status");
        if (timestamps_out && !io.timestamps)
            return fail(OB_INVALID_ARGUMENT, "timestamps_out requested without column timestamps");
        const ob_lut* lut = io.lut;
        if (lut->device != s->device) return fail(OB_INVALID_ARGUMENT, "lut and stream are on different devices");
        if (dtype < 0) dtype = lut->dtype;
        if (lut->dtype != dtype) return fail(OB_INVALID_ARGUMENT, "the luts of a set must share one dtype");
        if (lut->h == 0 || lut->w == 0) continue;
        K3Frame f;
        rs = stage_k3_frame(lut, io.range, io.poses, io.status, io.timestamps, timestamps_out != nullptr,
                            static_cast<unsigned>(i), stg, &f);
        if (rs != OB_OK) return rs;
        hf.push_back(f);
    }
    if (hf.empty()) return OB_OK;
    return run_dewarp(hf, dtype, min_r, max_r, points, capacity, frame_idx, col_idx, timestamps_out, counts, n_points,
                      stg, s);
}

ob_status ob_destagger(size_t elem_size, size_t k, const void* img, const int32_t* shifts,
                       size_t n_shifts, size_t h, size_t w, int inverse, void* out, ob_stream* s) {
    if (!s) return fail(OB_INVALID_ARGUMENT, "null stream");
    // checks and texts of destagger_into, impl/lidar_frame_impl.h:740-747
    if (n_shifts != h) return fail(OB_INVALID_ARGUMENT, "image height does not match shifts size");
    if (h == 0 || w == 0) return OB_OK;
    if (!img || !out || !shifts) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (elem_size == 0 || k == 0) return fail(OB_INVALID_ARGUMENT, "element size must be positive");
    if (w > 65535) return fail(OB_INVALID_ARGUMENT, "frame width exceeds 65535 columns");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    std::vector<uint16_t> sh;
    reduce_shifts(shifts, h, w, inverse, sh);
    const size_t bytes = h * w * k * elem_size;
    Staging stg(s->st);
    const void* din = nullptr;
    void* dout = nullptr;
    cudaError_t e = stg.in(img, bytes, &din);
    if (e != cudaSuccess) return fail_cuda(e, "stage image");
    e = stg.out(out, bytes, &dout);
    if (e != cudaSuccess) return fail_cuda(e, "stage output");
    if (din == dout) return fail(OB_INVALID_ARGUMENT, "image and destaggered must not alias");
    e = launch_destagger(elem_size, k, din, sh.data(), h, w, dout, s->device, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "destagger launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "destagger D2H");
    return OB_OK;
}

}  // extern "C"
