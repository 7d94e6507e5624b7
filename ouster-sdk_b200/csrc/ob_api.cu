// ob_api.cu -- C-ABI glue: error state, streams, staging of host buffers, LUT handles and the
// entry points declared in include/ouster_b200.h (everything except the decoder, decode and
// encode entry points, which live in ob_api_decode.cu).
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

static std::atomic<uint64_t> g_family[OB_FAM_COUNT];
static const char* const kFamilies[OB_FAM_COUNT] = {"decode_pipe", "decode", "cloud", "normals", "voxel",
                                                    "voxel_map", "icp", "align", "zone", "image",
                                                    "frame_ops", "pose", "dewarp", "destagger", "lut",
                                                    "encode", "ground"};

void record_launch(int family) {
    g_family[family].fetch_add(1, std::memory_order_relaxed);
    if (family == OB_FAM_DECODE_PIPE) g_family[OB_FAM_DECODE].fetch_add(1, std::memory_order_relaxed);
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
    // setting one of the plain K1 geometry tunables pins that geometry; cloud_auto = 1 gives the choice back
    if (n == "cloud_tw" || n == "cloud_stages" || n == "cloud_threads" || n == "cloud_ctas_per_sm") t.cloud_auto = 0;
    if (n == "cloud_auto") t.cloud_auto = value ? 1 : 0;
    else if (n == "cloud_tw") t.cloud_tw = std::max(4, value / 4 * 4);
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

void* Staging::stage(const void* p, size_t bytes, bool upload, bool download) {
    if (err_ != cudaSuccess) return nullptr;
    if (bytes == 0 || p == nullptr || is_device_ptr(p)) return const_cast<void*>(p);
    void* d = scratch_bytes(bytes);
    if (d && upload) check(cudaMemcpyAsync(d, p, bytes, cudaMemcpyHostToDevice, st_));
    if (d && download) pending_.push_back({const_cast<void*>(p), d, bytes, bytes, 1});
    return d;
}

void* Staging::out_rows(void* p, size_t row_bytes, size_t pitch, size_t rows) {
    if (err_ != cudaSuccess) return nullptr;
    if (row_bytes == 0 || rows == 0 || p == nullptr || is_device_ptr(p)) return p;
    void* d = scratch_bytes(row_bytes * rows);
    if (d) pending_.push_back({p, d, row_bytes, pitch, rows});
    return d;
}

void* Staging::scratch_bytes(size_t bytes) {
    if (err_ != cudaSuccess) return nullptr;
    void* d = nullptr;
    if (check(cudaMallocAsync(&d, bytes ? bytes : 16, st_)) != cudaSuccess) return nullptr;
    scratch_.push_back(d);
    return d;
}

cudaError_t Staging::flush() {
    for (const Pending& q : pending_) {
        if (err_ != cudaSuccess) break;
        check(q.rows == 1 ? cudaMemcpyAsync(q.host, q.dev, q.bytes, cudaMemcpyDeviceToHost, st_)
                          : cudaMemcpy2DAsync(q.host, q.pitch, q.dev, q.bytes, q.bytes, q.rows,
                                              cudaMemcpyDeviceToHost, st_));
    }
    pending_.clear();
    return err_;
}

cudaError_t Staging::finish() {
    const bool wait = !pending_.empty();
    if (flush() == cudaSuccess && wait) check(cudaStreamSynchronize(st_));
    return err_;
}

CountedRows::CountedRows(size_t* n, size_t capacity, Staging& stg, cudaStream_t st, const char* what)
    : n_(n), cap_(capacity), stg_(stg), st_(st), what_(what), dev_(is_device_ptr(n)) {
    if (n && !dev_) *n = 0;
}

ob_status CountedRows::zero() {
    if (!dev_ || zeroed_) return OB_OK;
    cudaError_t e = cudaMemsetAsync(n_, 0, sizeof(size_t), st_);
    if (e != cudaSuccess) return fail_cuda(e, what_);
    zeroed_ = true;
    return OB_OK;
}

ob_status CountedRows::refuse(std::initializer_list<const void*> arrays, const char* msg) {
    if (!dev_) return OB_OK;
    for (const void* p : arrays)
        if (p && !is_device_ptr(p)) {
            ob_status rs = zero();
            return rs != OB_OK ? rs : fail(OB_INVALID_ARGUMENT, msg);
        }
    return OB_OK;
}

void* CountedRows::array(void* p, size_t row_bytes) {
    if (stg_.error()) return nullptr;
    if (!p || is_device_ptr(p)) return p;
    void* d = stg_.scratch<void>(cap_ * row_bytes);
    if (d) host_.push_back({p, d, row_bytes});
    return d;
}

unsigned long long* CountedRows::word() {
    if (dev_) return reinterpret_cast<unsigned long long*>(n_);
    return stg_.scratch<unsigned long long>(1);
}

ob_status CountedRows::finish(const unsigned long long* end) {
    if (dev_) {
        if (end == reinterpret_cast<const unsigned long long*>(n_)) return OB_OK;  // the kernel wrote it in place
        cudaError_t e = cudaMemcpyAsync(n_, end, 8, cudaMemcpyDeviceToDevice, st_);
        return e == cudaSuccess ? OB_OK : fail_cuda(e, what_);
    }
    unsigned long long total = 0;
    ob_status rs = read(end, 1, &total);
    return rs != OB_OK ? rs : deliver(total);
}

ob_status CountedRows::read(const unsigned long long* ends, size_t k, unsigned long long* host) {
    cudaError_t e = cudaMemcpyAsync(host, ends, k * 8, cudaMemcpyDeviceToHost, st_);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st_);
    return e == cudaSuccess ? OB_OK : fail_cuda(e, what_);
}

ob_status CountedRows::deliver(unsigned long long total) {
    if (total > cap_) return fail(OB_INVALID_ARGUMENT, "output capacity too small");
    cudaError_t e = cudaSuccess;
    if (total && !host_.empty()) {
        for (const HostArray& a : host_)
            if (e == cudaSuccess) e = cudaMemcpyAsync(a.host, a.dev, total * a.row_bytes, cudaMemcpyDeviceToHost, st_);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st_);
    }
    if (e != cudaSuccess) return fail_cuda(e, what_);
    *n_ = static_cast<size_t>(total);
    return OB_OK;
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
        DeviceBlock dev;
        std::vector<uint8_t> host;
    } tables[3];
};

struct ob_lut {
    int device;
    int dtype;
    size_t h, w;
    DeviceBlock dir, off;
    // LUT-free mode (LUTs built from per-beam intrinsics only): device LutAnalyticT<T> + its tables
    DeviceBlock an, an_row, an_col;
    bool analytic_on{false};
};

namespace ob {
LutView lut_view(const ob_lut* lut) {
    return LutView{lut->dir.get(), lut->off.get(), lut->dtype, lut->h, lut->w, lut->device,
                   lut->analytic_on ? lut->an.get() : nullptr};
}
cudaStream_t stream_handle(ob_stream* s) { return s->st; }

cudaError_t stream_table(ob_stream* s, int which, const void* host, size_t bytes, const void** dev) {
    ob_stream::Table& t = s->tables[which];
    if (t.dev.get() && t.host.size() == bytes && std::memcmp(t.host.data(), host, bytes) == 0) {
        *dev = t.dev.get();  // identical to what the device already holds
        return cudaSuccess;
    }
    if (bytes > t.dev.bytes()) {
        if (t.dev.get()) {
            cudaError_t e = cudaStreamSynchronize(s->st);  // a running launch may still read the old table
            if (e != cudaSuccess) return e;
        }
        cudaError_t e = t.dev.alloc(std::max<size_t>(bytes * 2, 4096));
        if (e != cudaSuccess) return e;
    }
    t.host.assign(static_cast<const uint8_t*>(host), static_cast<const uint8_t*>(host) + bytes);
    // stream-ordered: lands after every earlier launch of this stream that reads the previous contents
    cudaError_t e = cudaMemcpyAsync(t.dev.get(), t.host.data(), bytes, cudaMemcpyHostToDevice, s->st);
    if (e != cudaSuccess) {
        t.host.clear();
        return e;
    }
    *dev = t.dev.get();
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
    if (n == "ob_image_params") return sizeof(ob_image_params);
    if (n == "ob_image_state") return sizeof(ob_image_state);
    if (n == "ob_frame_field") return sizeof(ob_frame_field);
    if (n == "ob_frame_ops_io") return sizeof(ob_frame_ops_io);
    if (n == "ob_frame_rows_entry") return sizeof(ob_frame_rows_entry);
    if (n == "ob_frame_rows_io") return sizeof(ob_frame_rows_io);
    if (n == "ob_map_rows") return sizeof(ob_map_rows);
    if (n == "ob_map_field") return sizeof(ob_map_field);
    if (n == "ob_map_rows_item") return sizeof(ob_map_rows_item);
    if (n == "ob_interp_pose_io") return sizeof(ob_interp_pose_io);
    if (n == "ob_frame_poses_item") return sizeof(ob_frame_poses_item);
    if (n == "ob_ground_model") return sizeof(ob_ground_model);
    if (n == "ob_ground_item") return sizeof(ob_ground_item);
    if (n == "ob_align_clouds_trace") return sizeof(ob_align_clouds_trace);
    if (n == "ob_align_clouds_io") return sizeof(ob_align_clouds_io);
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

uint64_t ob_kernel_launch_count(void) {
    uint64_t n = 0;
    for (int i = 0; i < OB_FAM_COUNT; ++i)
        if (i != OB_FAM_DECODE_PIPE) n += g_family[i].load(std::memory_order_relaxed);
    return n;
}

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
    DeviceScope on(s->device);
    bool have_tables = false;
    for (auto& t : s->tables) have_tables |= t.dev.get() != nullptr;
    if (s->owned || have_tables) cudaStreamSynchronize(s->st);
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
    DeviceBlock an, an_row, an_col;
    cudaError_t e = an_row.alloc(row.size() * sizeof(T));
    if (e == cudaSuccess) e = an_col.alloc(col.size() * sizeof(T));
    if (e == cudaSuccess) e = an.alloc(sizeof(a));
    if (e == cudaSuccess) e = cudaMemcpy(an_row.get(), row.data(), row.size() * sizeof(T), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(an_col.get(), col.data(), col.size() * sizeof(T), cudaMemcpyHostToDevice);
    a.row = an_row.get<const T>();
    a.col = an_col.get<const T>();
    if (e == cudaSuccess) e = cudaMemcpy(an.get(), &a, sizeof(a), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) return e;
    l->an = std::move(an);
    l->an_row = std::move(an_row);
    l->an_col = std::move(an_col);
    return cudaSuccess;
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
    std::unique_ptr<ob_lut> l(new ob_lut{device, static_cast<int>(dtype), h, w});
    cudaError_t e = l->dir.alloc(bytes);
    if (e == cudaSuccess) e = l->off.alloc(bytes);
    if (e != cudaSuccess) return fail_cuda(e, "cudaMalloc(lut)");
    e = cudaMemcpy(l->dir.get(), direction, bytes, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(l->off.get(), offset, bytes, cudaMemcpyDefault);
    if (e != cudaSuccess) return fail_cuda(e, "cudaMemcpy(lut)");
    *out = l.release();
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
    DeviceBlock dd, doff;  // the finished tables
    cudaError_t e;
    {  // the angles' device copies go before the LUT-free tables are allocated
        DeviceBlock daz, dalt;
        e = daz.alloc(n_az * 8);
        if (e == cudaSuccess) e = dalt.alloc(n_alt * 8);
        if (e == cudaSuccess) e = dd.alloc(n3 * 8);
        if (e == cudaSuccess) e = doff.alloc(n3 * 8);
        if (e == cudaSuccess) e = cudaMemcpy(daz.get(), az, n_az * 8, cudaMemcpyDefault);
        if (e == cudaSuccess) e = cudaMemcpy(dalt.get(), alt, n_alt * 8, cudaMemcpyDefault);
        if (e == cudaSuccess)
            e = launch_make_lut(w, h, range_unit, b2l, transform, daz.get<double>(), n_az, dalt.get<double>(), n_alt,
                                dd.get<double>(), doff.get<double>(), 0);
        if (e == cudaSuccess && dtype == OB_F32) {
            DeviceBlock fd, fo;
            e = fd.alloc(n3 * 4);
            if (e == cudaSuccess) e = fo.alloc(n3 * 4);
            if (e == cudaSuccess) e = launch_cast_f64_f32(dd.get<double>(), fd.get<float>(), n3, 0);
            if (e == cudaSuccess) e = launch_cast_f64_f32(doff.get<double>(), fo.get<float>(), n3, 0);
            if (e == cudaSuccess) e = cudaDeviceSynchronize();
            if (e == cudaSuccess) {
                dd = std::move(fd);
                doff = std::move(fo);
            }
        }
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    if (e != cudaSuccess) return fail_cuda(e, "ob_lut_from_intrinsics");
    ob_lut* l = new ob_lut{device, static_cast<int>(dtype), h, w, std::move(dd), std::move(doff)};
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
    if (enable && !lut->an.get())
        return fail(OB_INVALID_ARGUMENT, "LUT-free projection needs a lut built from per-beam intrinsics");
    lut->analytic_on = enable != 0;
    return OB_OK;
}

int ob_lut_is_analytic(const ob_lut* lut) { return lut && lut->analytic_on ? 1 : 0; }

ob_status ob_lut_download(const ob_lut* lut, void* direction, void* offset) {
    if (!lut || !direction || !offset) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const size_t bytes = lut->h * lut->w * 3 * dtype_size(lut->dtype);
    cudaSetDevice(lut->device);
    cudaError_t e = cudaMemcpy(direction, lut->dir.get(), bytes, cudaMemcpyDefault);
    if (e == cudaSuccess) e = cudaMemcpy(offset, lut->off.get(), bytes, cudaMemcpyDefault);
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
    if (direction) *direction = lut->dir.get();
    if (offset) *offset = lut->off.get();
    return OB_OK;
}

ob_status ob_lut_destroy(ob_lut* lut) {
    if (!lut) return OB_OK;
    DeviceScope on(lut->device);
    forget_lut_tensor_maps(lut->dir.get());
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
    // true when the [F][R][n] blocks tile their extent with no gap (frame- or return-major); a host output with
    // gaps is uploaded first, so that the copy back leaves the caller's bytes between the blocks as they were
    auto dense = [&](size_t fs, size_t rs, size_t n) {
        if (F > 1 && R > 1) return (rs == n && fs == R * n) || (fs == n && rs == F * n);
        if (R > 1) return rs == n;
        if (F > 1) return fs == n;
        return true;
    };
    auto stage_out = [&](auto* p, size_t fs, size_t rs, size_t n) {
        const size_t count = extent(fs, rs, n);
        return dense(fs, rs, n) ? stg.out(p, count) : stg.inout(p, count);
    };
    CloudArgs<T> a;
    a.dir = lut->dir.get<const T>();
    a.off = lut->off.get<const T>();
    a.analytic = lut->analytic_on ? lut->an.get<const LutAnalyticT<T>>() : nullptr;
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
    a.range = stg.in(io->range, extent(a.range_fs, a.range_rs, n_px));
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage range");
    a.xyz = nullptr;
    a.rd = nullptr;
    a.xd = nullptr;
    if (io->xyz) {
        a.xyz = stage_out(static_cast<T*>(io->xyz), a.xyz_fs, a.xyz_rs, n_px * 3);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage xyz");
    }
    if (io->range_destaggered) {
        a.rd = stage_out(io->range_destaggered, a.rd_fs, a.rd_rs, n_px);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage range_destaggered");
    }
    if (io->xyz_destaggered) {
        a.xd = stage_out(static_cast<T*>(io->xyz_destaggered), a.xd_fs, a.xd_rs, n_px * 3);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage xyz_destaggered");
    }
    if (io->poses) {
        const size_t pn = static_cast<size_t>(lut->w) * 16;
        a.poses = stg.in(static_cast<const T*>(io->poses), (F - 1) * io->poses_frame_stride + pn);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage poses");
        a.poses_fs = io->poses_frame_stride;
    }
    cudaError_t e = launch_cloud<T>(a, s->device, s->st);
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
    const void* dp = stg.in(points, n_points * 3 * esz);
    const void* dq = stg.in(poses, n_poses * 16 * esz);
    void* dout = stg.out(out, n_points * 3 * esz);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage dewarp buffers");
    const size_t H = n_points / n_poses;
    cudaError_t e;
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
// count (the per-frame ends of the look-back scan) through `res`.
static ob_status run_dewarp(std::vector<K3Frame>& hf, int dtype, uint32_t min_r, uint32_t max_r, void* points,
                            size_t capacity, uint32_t* frame_idx, uint32_t* col_idx, uint64_t* timestamps_out,
                            size_t* counts, CountedRows& res, Staging& stg, ob_stream* s) {
    unsigned n_blocks = 0, max_slabs = 0;
    for (K3Frame& f : hf) {
        f.first_block = n_blocks;
        n_blocks += f.n_cg;
        max_slabs = std::max(max_slabs, f.n_slabs);
    }
    const size_t esz = dtype_size(dtype);
    auto* fdev = stg.scratch<K3Frame>(hf.size());
    void* scan = stg.scratch<void>(dewarp_scan_scratch_bytes(n_blocks, static_cast<unsigned>(hf.size())));
    cudaError_t e = stg.error();
    if (e == cudaSuccess) e = cudaMemcpyAsync(fdev, hf.data(), hf.size() * sizeof(K3Frame), cudaMemcpyHostToDevice, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "frame table upload");
    void* dpts = res.array(points, 3 * esz);
    uint32_t* dfi = res.array(frame_idx, 4);
    uint32_t* dci = res.array(col_idx, 4);
    uint64_t* dts = res.array(timestamps_out, 8);
    e = stg.error();
    if (e != cudaSuccess) return fail_cuda(e, "stage dewarp outputs");
    const unsigned long long* fend = nullptr;
    e = launch_dewarp_fused(fdev, static_cast<unsigned>(hf.size()), n_blocks, max_slabs,
                            min_r, max_r, dtype, scan, dpts, dfi, dci, dts, capacity, &fend, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "dewarp launch");
    if (res.on_device()) return res.finish(fend + (hf.size() - 1));
    std::vector<unsigned long long> ends(hf.size());
    ob_status rs = res.read(fend, hf.size(), ends.data());
    if (rs == OB_OK) rs = res.deliver(ends.back());
    if (rs != OB_OK) return rs;  // counts keep their zeros, as *n_points does
    if (counts)
        for (size_t k = 0; k < hf.size(); ++k) counts[hf[k].index] = static_cast<size_t>(ends[k] - (k ? ends[k - 1] : 0ull));
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
    f.dir = lut->dir.get();
    f.off = lut->off.get();
    const size_t n_px = lut->h * lut->w;
    f.range = stg.in(range, n_px);
    f.poses = stg.in(poses, lut->w * 16);
    f.status = stg.in(status, lut->w);
    if (want_ts) f.timestamps = stg.in(timestamps, lut->w);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage dewarp inputs");
    *out = f;
    return OB_OK;
}

// The reference's window in millimetres, static_cast<uint32_t>(ceil(min_range * 1e3)) and the same with floor for
// max_range (dewarp_impl.h:34-35).  That cast is undefined unless the value lies in [0, 2^32), so a bound outside
// [0, 4294967295] mm, infinite or NaN is refused; ceil's -0.0 converts to 0.
static ob_status range_window(double min_range, double max_range, uint32_t* min_r, uint32_t* max_r) {
    const double lo = std::ceil(min_range * 1e3), hi = std::floor(max_range * 1e3);
    if (!(lo >= 0.0 && lo <= 4294967295.0 && hi >= 0.0 && hi <= 4294967295.0))
        return fail(OB_INVALID_ARGUMENT, "range window outside [0, 4294967.295] m: ceil(min_range * 1e3) and "
                                         "floor(max_range * 1e3) must lie in [0, 4294967295] mm");
    *min_r = static_cast<uint32_t>(lo);
    *max_r = static_cast<uint32_t>(hi);
    return OB_OK;
}

static const char* const kDewarpMixed = "a device-side count needs device outputs and no per-frame counts";
static const char* const kDewarpRows = "dewarp supports at most 25600 rows per frame";

ob_status ob_dewarp_frame(const ob_lut* lut, const ob_dewarp_frame_io* io, size_t* n_points, ob_stream* s) {
    if (!lut || !io || !n_points || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    Staging stg(s->st);
    CountedRows res(n_points, io->capacity, stg, s->st, "dewarp count");
    rs = res.zero();
    if (rs != OB_OK) return rs;
    if (!io->range || !io->poses || !io->status || !io->points)
        return fail(OB_INVALID_ARGUMENT, "null range / poses / status / points");
    if (io->timestamps_out && !io->timestamps)
        return fail(OB_INVALID_ARGUMENT, "timestamps_out requested without column timestamps");
    if (lut->device != s->device) return fail(OB_INVALID_ARGUMENT, "lut and stream are on different devices");
    if (lut->h > kDewarpMaxRows) return fail(OB_INVALID_ARGUMENT, kDewarpRows);
    uint32_t min_r, max_r;
    rs = range_window(io->min_range, io->max_range, &min_r, &max_r);
    if (rs != OB_OK) return rs;
    if (min_r > max_r || lut->h == 0 || lut->w == 0) return OB_OK;
    rs = res.refuse({io->points, io->col_idx, io->timestamps_out}, kDewarpMixed);
    if (rs != OB_OK) return rs;
    std::vector<K3Frame> hf(1);
    rs = stage_k3_frame(lut, io->range, io->poses, io->status, io->timestamps, io->timestamps_out != nullptr, 0, stg, &hf[0]);
    if (rs != OB_OK) return rs;
    return run_dewarp(hf, lut->dtype, min_r, max_r, io->points, io->capacity, nullptr, io->col_idx, io->timestamps_out,
                      nullptr, res, stg, s);
}

ob_status ob_dewarp_frames(const ob_dewarp_frames_io* frames, size_t n_frames, double min_range, double max_range,
                           void* points, size_t capacity, uint32_t* frame_idx, uint32_t* col_idx,
                           uint64_t* timestamps_out, size_t* counts, size_t* n_points, ob_stream* s) {
    if (!s || !n_points || (n_frames && !frames)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    ob_status rs = require_device(s->device);
    if (rs != OB_OK) return rs;
    Staging stg(s->st);
    CountedRows res(n_points, capacity, stg, s->st, "dewarp count");
    rs = res.zero();
    if (rs != OB_OK) return rs;
    if (counts) std::fill(counts, counts + n_frames, static_cast<size_t>(0));
    if (n_frames == 0) return OB_OK;
    if (!points) return fail(OB_INVALID_ARGUMENT, "null points buffer");
    uint32_t min_r, max_r;
    rs = range_window(min_range, max_range, &min_r, &max_r);
    if (rs != OB_OK) return rs;
    int dtype = -1;
    std::vector<size_t> live;  // frames with pixels, checked before any is staged
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
        if (lut->h > kDewarpMaxRows) return fail(OB_INVALID_ARGUMENT, kDewarpRows);
        if (lut->h != 0 && lut->w != 0) live.push_back(i);
    }
    if (min_r > max_r || live.empty()) return OB_OK;
    rs = res.refuse({points, frame_idx, col_idx, timestamps_out, counts}, kDewarpMixed);
    if (rs != OB_OK) return rs;
    std::vector<K3Frame> hf(live.size());
    for (size_t k = 0; k < live.size(); ++k) {
        const ob_dewarp_frames_io& io = frames[live[k]];
        rs = stage_k3_frame(io.lut, io.range, io.poses, io.status, io.timestamps, timestamps_out != nullptr,
                            static_cast<unsigned>(live[k]), stg, &hf[k]);
        if (rs != OB_OK) return rs;
    }
    return run_dewarp(hf, dtype, min_r, max_r, points, capacity, frame_idx, col_idx, timestamps_out, counts, res, stg,
                      s);
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
    const void* din = stg.in(img, bytes);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage image");
    void* dout = stg.out(out, bytes);
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage output");
    if (din == dout) return fail(OB_INVALID_ARGUMENT, "image and destaggered must not alias");
    cudaError_t e = launch_destagger(elem_size, k, din, sh.data(), h, w, dout, s->device, s->st);
    if (e != cudaSuccess) return fail_cuda(e, "destagger launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "destagger D2H");
    return OB_OK;
}

}  // extern "C"
