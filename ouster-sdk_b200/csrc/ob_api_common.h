// ob_api_common.h -- helpers shared by the C-ABI translation units.
#pragma once
#include <string>
#include <vector>

#include "ob_internal.h"

namespace ob {

ob_status fail(ob_status st, const std::string& msg);
ob_status fail_cuda(cudaError_t e, const char* what);
ob_status require_device(int device);
bool is_device_ptr(const void* p);
void reduce_shifts(const int32_t* shifts, size_t h, size_t w, int inverse, std::vector<uint16_t>& out);

// Per-call staging of host buffers through stream-ordered device scratch.
// in():  host -> scratch (H2D issued immediately); device pointers pass through.
// out(): scratch now, D2H issued by flush() after the kernel; device pointers pass through.
// inout(): as out(), but the host contents are uploaded first, so bytes the kernel leaves alone
//          (padding between strided frames) come back unchanged.
class Staging {
   public:
    explicit Staging(cudaStream_t st) : st_(st) {}
    ~Staging();
    cudaError_t in(const void* p, size_t bytes, const void** dev);
    cudaError_t out(void* p, size_t bytes, void** dev);
    cudaError_t inout(void* p, size_t bytes, void** dev);
    cudaError_t scratch(size_t bytes, void** dev);
    cudaError_t flush();

   private:
    struct Pending {
        void* host;
        void* dev;
        size_t bytes;
    };
    cudaStream_t st_;
    std::vector<void*> scratch_;
    std::vector<Pending> pending_;
};

// accessors for the opaque handles (defined in ob_api.cu)
void lut_view(const ob_lut* lut, const void** dir, const void** off, int* dtype, size_t* h,
              size_t* w, int* device);
const void* lut_analytic(const ob_lut* lut);  // device LutAnalyticT<T> when the LUT-free mode is on, else null
cudaStream_t stream_handle(ob_stream* s);
// device copy of a small per-launch table (which: 0 decode frames, 1 encode frames), re-uploaded only when
// its contents changed since the stream's previous launch of that kind
cudaError_t stream_table(ob_stream* s, int which, const void* host, size_t bytes, const void** dev);
int stream_device(ob_stream* s);

}  // namespace ob
