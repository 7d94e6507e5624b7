// ob_api_common.h -- helpers shared by the C-ABI translation units.
#pragma once
#include <initializer_list>
#include <memory>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "ob_internal.h"

namespace ob {

ob_status fail(ob_status st, const std::string& msg);
ob_status fail_cuda(cudaError_t e, const char* what);
ob_status require_device(int device);
bool is_device_ptr(const void* p);
void reduce_shifts(const int32_t* shifts, size_t h, size_t w, int inverse, std::vector<uint16_t>& out);

// Per-call staging of host buffers through stream-ordered device scratch.  Sizes count elements of T (bytes when T
// is void); a null pointer, a device pointer or a zero-size request is returned as is.
// in():  host -> scratch (H2D issued immediately).
// out(): scratch now, D2H issued by flush() after the kernel.
// inout(): as out(), but the host contents are uploaded first, so bytes the kernel leaves alone
//          (padding between strided frames) come back unchanged.
// out_rows(): out() for `rows` blocks of `row_bytes` that lie `pitch` bytes apart on the host.  The scratch holds
//          them back to back and flush() copies each block to its place: host bytes between the blocks are
//          neither read nor written.
// scratch(): device memory for the call, freed in stream order when the Staging goes (at least 16 bytes).
// The first CUDA error of the call is kept: error() returns it, and from then on in / out / inout / scratch return
// null and make no CUDA call, and flush() / finish() return it.  check() records an error met outside the Staging.
class Staging {
   public:
    explicit Staging(cudaStream_t st) : st_(st) {}
    ~Staging();
    cudaError_t error() const { return err_; }
    cudaError_t check(cudaError_t e) {
        if (err_ == cudaSuccess) err_ = e;
        return err_;
    }
    template <typename T>
    const T* in(const T* p, size_t n) {
        return static_cast<const T*>(stage(p, n * elem_bytes<T>(), true, false));
    }
    template <typename T>
    T* out(T* p, size_t n) {
        return static_cast<T*>(stage(p, n * elem_bytes<T>(), false, true));
    }
    template <typename T>
    T* inout(T* p, size_t n) {
        return static_cast<T*>(stage(p, n * elem_bytes<T>(), true, true));
    }
    void* out_rows(void* p, size_t row_bytes, size_t pitch, size_t rows);
    template <typename T>
    T* scratch(size_t n) {
        return static_cast<T*>(scratch_bytes(n * elem_bytes<T>()));
    }
    cudaError_t flush();
    // flush(), then wait for the stream if that issued a D2H: host results are final on return, and a call whose
    // outputs are all device memory waits for nothing (and stays capturable in a CUDA graph)
    cudaError_t finish();

   private:
    template <typename T>
    static constexpr size_t elem_bytes() {
        if constexpr (std::is_void_v<T>) return 1;
        else return sizeof(T);
    }
    // scratch for a host buffer, filled from it (upload) and copied back to it by flush() (download)
    void* stage(const void* p, size_t bytes, bool upload, bool download);
    void* scratch_bytes(size_t bytes);
    struct Pending {  // `rows` blocks of `bytes`, dense on the device, `pitch` apart on the host
        void* host;
        void* dev;
        size_t bytes;
        size_t pitch;
        size_t rows;
    };
    cudaStream_t st_;
    cudaError_t err_ = cudaSuccess;
    std::vector<void*> scratch_;
    std::vector<Pending> pending_;
};

// Memory a handle keeps across calls: one cudaMalloc block (cudaHostAlloc when Pinned) and its size, freed when the
// owner goes or takes another block.  Move-only.  Frees are not stream-ordered: cudaFree waits for the device.
template <bool Pinned>
class Block {
   public:
    Block() = default;
    Block(Block&& o) noexcept : p_(std::exchange(o.p_, nullptr)), bytes_(std::exchange(o.bytes_, 0)) {}
    Block& operator=(Block&& o) noexcept {
        if (this != &o) {
            release();
            p_ = std::exchange(o.p_, nullptr);
            bytes_ = std::exchange(o.bytes_, 0);
        }
        return *this;
    }
    ~Block() { release(); }
    // frees the block, then allocates one of `bytes`; on failure the owner is left empty
    cudaError_t alloc(size_t bytes) {
        release();
        void* p = nullptr;
        cudaError_t e = Pinned ? cudaHostAlloc(&p, bytes, cudaHostAllocDefault) : cudaMalloc(&p, bytes);
        if (e == cudaSuccess) {
            p_ = p;
            bytes_ = bytes;
        }
        return e;
    }
    // alloc(bytes) unless the block already has that many; the contents are not kept
    cudaError_t reserve(size_t bytes) { return bytes <= bytes_ ? cudaSuccess : alloc(bytes); }
    template <typename T = void>
    T* get() const {
        return static_cast<T*>(p_);
    }
    size_t bytes() const { return bytes_; }

   private:
    void release() {
        if (p_) Pinned ? cudaFreeHost(p_) : cudaFree(p_);
        p_ = nullptr;
        bytes_ = 0;
    }
    void* p_ = nullptr;
    size_t bytes_ = 0;
};
using DeviceBlock = Block<false>;
using PinnedBlock = Block<true>;

// A cudaEvent_t (timing disabled) a handle keeps across calls, destroyed with its owner.
class Event {
   public:
    Event() = default;
    Event(const Event&) = delete;
    Event& operator=(const Event&) = delete;
    ~Event() {
        if (ev_) cudaEventDestroy(ev_);
    }
    cudaError_t create() { return cudaEventCreateWithFlags(&ev_, cudaEventDisableTiming); }
    cudaEvent_t get() const { return ev_; }

   private:
    cudaEvent_t ev_ = nullptr;
};

// Makes `device` current for the scope and gives the caller's current device back when it ends.
class DeviceScope {
   public:
    explicit DeviceScope(int device) {
        cudaGetDevice(&prev_);
        cudaSetDevice(device);
    }
    ~DeviceScope() { cudaSetDevice(prev_); }
    DeviceScope(const DeviceScope&) = delete;
    DeviceScope& operator=(const DeviceScope&) = delete;

   private:
    int prev_ = 0;
};

// A result whose length the GPU decides: rows in one or more arrays plus their count, each in host or device memory.
//  - The count reads 0 until the call succeeds: a host count is zeroed here, a device count by zero() (or by the
//    kernel that writes it).
//  - A device count needs every array in device memory; refuse() turns a host array away (count 0) before anything
//    is staged or launched.
//  - array(): a device array is written in place, a host array through scratch of `capacity` rows, a null array is
//    not written (count only).  array() and word() allocate through the call's Staging and return null after an error.
//  - finish(): with a device count nothing waits, rows past `capacity` are cut and the count is the true total.  With
//    a host count the call waits for the count; more rows than `capacity` fail "output capacity too small" with the
//    count left 0 and the host rows untouched; otherwise it waits again for the rows of the host arrays.
class CountedRows {
   public:
    static constexpr size_t kCountOnly = ~static_cast<size_t>(0);  // capacity of a call that writes no rows
    CountedRows(size_t* n, size_t capacity, Staging& stg, cudaStream_t st, const char* what);
    bool on_device() const { return dev_; }
    ob_status zero();
    ob_status refuse(std::initializer_list<const void*> arrays, const char* msg);
    void* array(void* p, size_t row_bytes);
    template <typename T>
    T* array(T* p, size_t row_bytes) {
        return static_cast<T*>(array(static_cast<void*>(p), row_bytes));
    }
    // the device word the kernel writes the count to: the caller's device count, or scratch
    unsigned long long* word();
    // after the launch; `end`: the device word holding the count
    ob_status finish(const unsigned long long* end);
    // finish() in two steps for a host count: read k device words (the last is the count) with one wait, then deliver
    ob_status read(const unsigned long long* ends, size_t k, unsigned long long* host);
    ob_status deliver(unsigned long long total);

   private:
    struct HostArray {
        void* host;
        void* dev;
        size_t row_bytes;
    };
    size_t* n_;
    size_t cap_;
    Staging& stg_;
    cudaStream_t st_;
    const char* what_;
    bool dev_, zeroed_ = false;
    std::vector<HostArray> host_;
};

// accessors for the opaque handles (defined in ob_api.cu)
struct LutView {
    const void* dir;
    const void* off;
    int dtype;
    size_t h, w;
    int device;
    const void* an;  // device LutAnalyticT<T> when the LUT-free mode is on, else null
};
LutView lut_view(const ob_lut* lut);
cudaStream_t stream_handle(ob_stream* s);
// device copy of a small per-launch table (which: 0 decode frames, 1 encode frames, 2 pose frames), re-uploaded only when
// its contents changed since the stream's previous launch of that kind
cudaError_t stream_table(ob_stream* s, int which, const void* host, size_t bytes, const void** dev);
int stream_device(ob_stream* s);

}  // namespace ob
