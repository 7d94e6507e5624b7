// ob_api_decode.cu -- C-ABI glue of the packet decode and encode: ob_decoder_*, the three decode entry points
// (ob_decode_frames, ob_decode_batch_run, ob_decode_job_*) and ob_encode_frames.
#include <algorithm>
#include <cstring>
#include <memory>
#include <vector>

#include "ob_api_common.h"
#include "ob_encode.h"

using namespace ob;

struct ob_decoder {
    int device;
    DecodeLayout L;
};

static bool valid_elem_size(uint32_t es) { return es == 1 || es == 2 || es == 4 || es == 8 || es == 6; }

static DecodeField to_dev(const ob_field_desc& f) {
    DecodeField d;
    d.offset = f.offset;
    d.elem_size = f.elem_size;
    d.mask = f.mask;
    d.shift = f.shift;
    d.range_return = f.range_return;
    d.zero_pattern = f.zero_pattern;
    d.pad = 0;
    return d;
}

// Frames of independent sensor streams carry their own LUTs.  The frame table is only a work list
// (every entry holds its own output pointers), so it may be reordered freely: keeping the frames
// of one LUT together lets each 6-12 MB table stay L2-resident while its frames are processed.
static void group_by_lut(std::vector<DecodeFrame>& frames) {
    bool any = false;
    for (const DecodeFrame& f : frames) any |= f.lut_dir != nullptr;
    if (!any) return;
    std::stable_sort(frames.begin(), frames.end(), [](const DecodeFrame& a, const DecodeFrame& b) {
        return reinterpret_cast<uintptr_t>(a.lut_dir) < reinterpret_cast<uintptr_t>(b.lut_dir);
    });
}

// TMA descriptors of a LUT for the pipelined K2 (null: that kernel is not applicable / not available)
static const void* maps_for(const DecodeLayout& L, int device, const void* dir, const void* off, int dtype) {
    uint32_t bw = 0, bh = 0;
    if (!dir || !off || !decode_pipe_box(L, device, dtype, &bw, &bh)) return nullptr;
    return lut_tensor_maps(dir, off, dtype, L.H, L.W, bw, bh, device);
}

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

constexpr size_t kMaxSlots = size_t(1) << 20;  // packet slots of one frame

// The outputs of a decoded frame in one numbering: field k < OB_MAX_FIELDS, the three column headers, then XYZ and
// destaggered range of each return (the order in which the paths stage them)
enum : int { kOutTs = OB_MAX_FIELDS, kOutMid, kOutStatus, kOutReturns, kOuts = kOutReturns + 2 * OB_MAX_RETURNS };
static bool is_xyz(int k) { return k >= kOutReturns && (k - kOutReturns) % 2 == 0; }

// bytes of output k of one frame (XYZ in the call's LUT dtype)
static size_t out_bytes(const DecodeLayout& L, int dtype, int k) {
    const size_t n_px = static_cast<size_t>(L.H) * L.W;
    if (k < kOutTs) return n_px * L.fields[k].elem_size;
    if (k == kOutTs) return L.W * 8ull;
    if (k == kOutMid) return L.W * 2ull;
    if (k == kOutStatus) return L.W * 4ull;
    return is_xyz(k) ? n_px * 3 * (dtype == OB_F64 ? 8 : 4) : n_px * 4;
}

// output k of an ob_decode_io, or of frame 0 of an ob_decode_batch; null: not requested
template <typename IO>
static void* io_out(const DecodeLayout& L, const IO& io, int k) {
    if (k < kOutTs) return k < static_cast<int>(L.n_fields) ? io.fields[k] : nullptr;
    if (k == kOutTs) return io.timestamp;
    if (k == kOutMid) return io.measurement_id;
    if (k == kOutStatus) return io.status;
    const int r = (k - kOutReturns) / 2;
    return is_xyz(k) ? io.xyz[r] : io.range_destaggered[r];
}

// bytes from a batch frame's output k to the next frame's
static size_t batch_stride(const ob_decode_batch& b, int k) {
    if (k < kOutTs) return b.field_frame_stride[k];
    if (k == kOutTs) return b.timestamp_frame_stride;
    if (k == kOutMid) return b.measurement_id_frame_stride;
    if (k == kOutStatus) return b.status_frame_stride;
    return is_xyz(k) ? b.xyz_frame_stride : b.rd_frame_stride;
}

static void set_out(DecodeFrame& f, int k, void* p) {
    const int r = (k - kOutReturns) / 2;
    if (k < kOutTs) f.fields[k] = p;
    else if (k == kOutTs) f.timestamp = static_cast<uint64_t*>(p);
    else if (k == kOutMid) f.measurement_id = static_cast<uint16_t*>(p);
    else if (k == kOutStatus) f.status = static_cast<uint32_t*>(p);
    else if (is_xyz(k)) f.xyz[r] = p;
    else f.rd[r] = static_cast<uint32_t*>(p);
}

// A LUT of a decode call as the kernels see it
struct CallLut {
    const void* dir{nullptr};
    const void* off{nullptr};
    const void* maps{nullptr};  // TMA descriptors for the pipelined kernel, or null
    const void* an{nullptr};    // LUT-free mode, or null
};

// One decode call: its checked arguments, and the launch-level facts every frame of its table folds into
struct DecodeCall {
    const DecodeLayout* L;
    int device;
    const ob_lut* lut;         // call-level LUT (nullable) ...
    CallLut call_lut;          // ... as the kernels see it
    int dtype{OB_F32};         // the one dtype of every LUT of the call
    int n_luts{0};
    std::vector<uint16_t> sh;  // shift table reduced to [0, W); empty: no shifts
    bool vec_ok{true}, frame_luts_have_maps{true}, any_xyz{false};
};

static ob_status same_device(const ob_decoder* dec, ob_stream* s) {
    if (stream_device(s) != dec->device) return fail(OB_INVALID_ARGUMENT, "decoder and stream are on different devices");
    return OB_OK;
}

// Checks a LUT of the call, call-level or per-frame: every LUT of one launch has the decoder's shape, the call's
// device and one dtype, because the kernel is instantiated for one dtype and XYZ outputs are sized by it
static ob_status take_lut(DecodeCall& c, const ob_lut* lut, CallLut* out) {
    const LutView v = lut_view(lut);
    if (v.h != c.L->H || v.w != c.L->W) return fail(OB_INVALID_ARGUMENT, "unexpected image dimensions");
    if (v.device != c.device) return fail(OB_INVALID_ARGUMENT, "lut and stream are on different devices");
    if (c.n_luts++ > 0 && v.dtype != c.dtype)
        return fail(OB_INVALID_ARGUMENT,
                    c.lut ? "per-frame lut dtype differs from the call-level lut" : "per-frame lut dtype differs");
    c.dtype = v.dtype;
    if (!al16(v.dir) || !al16(v.off)) c.vec_ok = false;
    *out = CallLut{v.dir, v.off, maps_for(*c.L, c.device, v.dir, v.off, v.dtype), v.an};
    return OB_OK;
}

// The start of every decode call: device, call-level LUT and shift table
static ob_status begin_call(DecodeCall& c, const ob_decoder* dec, ob_stream* s, const ob_lut* lut,
                            const int32_t* shifts, size_t n_shifts) {
    ob_status rs = same_device(dec, s);
    if (rs == OB_OK) rs = require_device(dec->device);
    if (rs != OB_OK) return rs;
    const DecodeLayout& L = dec->L;
    c.L = &L;
    c.device = dec->device;
    c.lut = lut;
    if (lut && (rs = take_lut(c, lut, &c.call_lut)) != OB_OK) return rs;
    if (shifts) {
        if (n_shifts != L.H) return fail(OB_INVALID_ARGUMENT, "image height does not match shifts size");
        if (L.H > static_cast<uint32_t>(kMaxRows))
            return fail(OB_INVALID_ARGUMENT, "fused destagger supports at most 512 rows");
        reduce_shifts(shifts, L.H, L.W, 0, c.sh);
    }
    return OB_OK;
}

// XYZ needs a LUT, destaggered range a shift table
static ob_status check_fused(const DecodeCall& c, bool has_lut, void* const xyz[], uint32_t* const rd[]) {
    for (int r = 0; r < OB_MAX_RETURNS; ++r) {
        if (xyz[r] && !has_lut) return fail(OB_INVALID_ARGUMENT, "xyz output requested without a lut");
        if (rd[r] && c.sh.empty()) return fail(OB_INVALID_ARGUMENT, "image height does not match shifts size");
    }
    return OB_OK;
}

// Sets a frame's flag bits and its own LUT (null: the call-level one) once its packets, column map and outputs are
// in place, and folds the frame into the launch-level facts
static void finish_frame(DecodeCall& c, DecodeFrame& f, bool bulk_ok, const CallLut* lut) {
    bool all_fields = c.L->n_fields > 0;
    for (uint32_t k = 0; k < c.L->n_fields; ++k) all_fields = all_fields && f.fields[k] != nullptr;
    f.flags = (f.col_src ? 0u : kFrameIdentityMap) | (bulk_ok ? kFrameBulkPackets : 0u) |
              (all_fields ? kFrameAllFields : 0u);
    if (lut) {
        f.lut_dir = lut->dir;
        f.lut_off = lut->off;
        f.lut_maps = lut->maps;
        f.lut_an = lut->an;
        if (!lut->maps && !lut->an) c.frame_luts_have_maps = false;
    }
    for (int r = 0; r < OB_MAX_RETURNS; ++r) {
        if (!f.xyz[r]) continue;
        c.any_xyz = true;
        if (!al16(f.xyz[r])) c.vec_ok = false;
    }
}

// xyz_base / xyz_frame_stride: the XYZ outputs of a uniformly strided batch (frame f at base + f * stride)
static cudaError_t launch(const DecodeCall& c, const void* frames_dev, size_t n_frames, cudaStream_t st,
                          const void* const* xyz_base = nullptr, unsigned long long xyz_frame_stride = 0) {
    DecodeLaunch a;
    a.layout_host = c.L;
    a.frames_dev = static_cast<const DecodeFrame*>(frames_dev);
    a.n_frames = static_cast<uint32_t>(n_frames);
    a.lut_dir = c.call_lut.dir;
    a.lut_off = c.call_lut.off;
    a.lut_dtype = c.dtype;
    a.shift_host = c.sh.empty() ? nullptr : c.sh.data();
    a.vec_ok = c.vec_ok;
    a.lut_maps = c.call_lut.maps;
    a.lut_an = c.call_lut.an;
    a.frame_luts_have_maps = c.frame_luts_have_maps;
    a.any_xyz = c.any_xyz;
    if (xyz_base) {
        a.xyz_base[0] = xyz_base[0];
        a.xyz_base[1] = xyz_base[1];
        a.xyz_frame_stride = xyz_frame_stride;
    }
    return launch_decode(a, c.device, st);
}

// ob_decode_frames and ob_decode_batch_run: the table goes through the stream's cached copy, host outputs come
// back from their staging after the launch
static ob_status run_table(const DecodeCall& c, ob_stream* s, std::vector<DecodeFrame>& hf, Staging& stg,
                           const void* const* xyz_base = nullptr, unsigned long long xyz_frame_stride = 0) {
    group_by_lut(hf);
    const void* fdev = nullptr;
    cudaError_t e = stream_table(s, 0, hf.data(), hf.size() * sizeof(DecodeFrame), &fdev);
    if (e != cudaSuccess) return fail_cuda(e, "frame table upload");
    e = launch(c, fdev, hf.size(), stream_handle(s), xyz_base, xyz_frame_stride);
    if (e != cudaSuccess) return fail_cuda(e, "decode launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "decode D2H");
    return OB_OK;
}

extern "C" {

ob_status ob_decoder_create(const ob_packet_layout* layout, const ob_field_desc* fields,
                            size_t n_fields, int device, ob_decoder** out) {
    if (!layout || !out || (n_fields && !fields)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (n_fields > OB_MAX_FIELDS) return fail(OB_INVALID_ARGUMENT, "too many fields");
    if (layout->columns_per_packet == 0)
        return fail(OB_INVALID_ARGUMENT, "unexpected columns_per_packet: 0");  // lidar_frame.cpp:1250-1252
    if (layout->pixels_per_column == 0)
        return fail(OB_INVALID_ARGUMENT, "unexpected pixels_per_column: 0");   // lidar_frame.cpp:1253-1255
    if (layout->columns_per_frame == 0) return fail(OB_INVALID_ARGUMENT, "unexpected frame dimensions");
    if (layout->columns_per_packet > 64)
        return fail(OB_INVALID_ARGUMENT, "columns_per_packet above 64 is not supported");
    if (layout->packet_size > 65535)
        return fail(OB_INVALID_ARGUMENT, "lidar_packet_size cannot exceed 65535");  // parsing.cpp:471-473
    const uint64_t need = static_cast<uint64_t>(layout->packet_header_size) +
                          static_cast<uint64_t>(layout->columns_per_packet) * layout->col_size;
    if (need > layout->packet_size ||
        static_cast<uint64_t>(layout->col_header_size) +
                static_cast<uint64_t>(layout->pixels_per_column) * layout->channel_data_size >
            layout->col_size)
        return fail(OB_INVALID_ARGUMENT, "inconsistent packet layout");
    for (size_t i = 0; i < n_fields; ++i) {
        if (!valid_elem_size(fields[i].elem_size))
            return fail(OB_INVALID_ARGUMENT, "Dest type too small for specified field");
        if (fields[i].offset >= layout->channel_data_size + 8u && layout->channel_data_size > 0)
            return fail(OB_INVALID_ARGUMENT, "field offset outside the channel data block");
        if (fields[i].range_return >= OB_MAX_RETURNS)
            return fail(OB_INVALID_ARGUMENT, "range_return must be < 2");
        if (fields[i].range_return >= 0 && fields[i].elem_size != 4)
            return fail(OB_INVALID_ARGUMENT, "range fields must decode to uint32");
    }
    ob_status rs = require_device(device);
    if (rs != OB_OK) return rs;
    ob_decoder* d = new ob_decoder;
    d->device = device;
    std::memset(&d->L, 0, sizeof(d->L));
    d->L.packet_header_size = layout->packet_header_size;
    d->L.col_header_size = layout->col_header_size;
    d->L.channel_data_size = layout->channel_data_size;
    d->L.col_size = layout->col_size;
    d->L.packet_size = layout->packet_size;
    d->L.cpp = layout->columns_per_packet;
    d->L.H = layout->pixels_per_column;
    d->L.W = layout->columns_per_frame;
    d->L.ts = to_dev(layout->col_timestamp);
    d->L.mid = to_dev(layout->col_measurement_id);
    d->L.status = to_dev(layout->col_status);
    d->L.n_fields = static_cast<uint32_t>(n_fields);
    for (size_t i = 0; i < n_fields; ++i) d->L.fields[i] = to_dev(fields[i]);
    *out = d;
    return OB_OK;
}

ob_status ob_decoder_destroy(ob_decoder* dec) {
    delete dec;
    return OB_OK;
}

ob_status ob_decode_frames(const ob_decoder* dec, const ob_decode_io* frames, size_t n_frames,
                           const ob_lut* lut, const int32_t* shifts, size_t n_shifts, ob_stream* s) {
    if (!dec || !s || (n_frames && !frames)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (n_frames == 0) return OB_OK;
    DecodeCall c;
    ob_status rs = begin_call(c, dec, s, lut, shifts, n_shifts);
    if (rs != OB_OK) return rs;
    const DecodeLayout& L = dec->L;
    Staging stg(stream_handle(s));
    std::vector<DecodeFrame> hf(n_frames);
    for (size_t i = 0; i < n_frames; ++i) {
        const ob_decode_io& io = frames[i];
        DecodeFrame& f = hf[i];
        std::memset(&f, 0, sizeof(f));
        if (io.n_slots > 0 && !io.packets) return fail(OB_INVALID_ARGUMENT, "null packet buffer");
        if (io.n_slots > 0 && io.packet_stride < L.packet_size)
            return fail(OB_INVALID_ARGUMENT, "packet_stride smaller than the lidar packet size");
        if (io.n_slots > kMaxSlots) return fail(OB_INVALID_ARGUMENT, "too many packet slots");
        CallLut frame_lut;
        if (io.lut && (rs = take_lut(c, io.lut, &frame_lut)) != OB_OK) return rs;
        if ((rs = check_fused(c, lut || io.lut, io.xyz, io.range_destaggered)) != OB_OK) return rs;
        if (io.n_slots > 0) {
            f.packets = stg.in(io.packets, (io.n_slots - 1) * io.packet_stride + L.packet_size);
            if (cudaError_t e = stg.error()) return fail_cuda(e, "stage packets");
        }
        f.packet_stride = io.packet_stride;
        f.n_slots = static_cast<uint32_t>(io.n_slots);
        if (io.col_src) {
            f.col_src = stg.in(io.col_src, L.W);
            if (cudaError_t e = stg.error()) return fail_cuda(e, "stage column map");
        }
        for (int k = 0; k < kOuts; ++k) {
            void* user = io_out(L, io, k);
            if (!user) continue;
            set_out(f, k, stg.out(user, out_bytes(L, c.dtype, k)));
            if (cudaError_t e = stg.error()) return fail_cuda(e, "stage outputs");
        }
        const bool bulk_ok = f.packets && al16(f.packets) && io.packet_stride % 16 == 0 && L.packet_size % 16 == 0;
        finish_frame(c, f, bulk_ok, io.lut ? &frame_lut : nullptr);
    }
    return run_table(c, s, hf, stg);
}

ob_status ob_decode_batch_run(const ob_decoder* dec, const ob_decode_batch* b, const ob_lut* lut,
                              const int32_t* shifts, size_t n_shifts, ob_stream* s) {
    if (!dec || !b || !s) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (b->n_frames == 0) return OB_OK;
    DecodeCall c;
    ob_status rs = begin_call(c, dec, s, lut, shifts, n_shifts);
    if (rs != OB_OK) return rs;
    const DecodeLayout& L = dec->L;
    if (!b->packets || b->n_slots == 0) return fail(OB_INVALID_ARGUMENT, "null packet buffer");
    if (b->packet_stride < L.packet_size)
        return fail(OB_INVALID_ARGUMENT, "packet_stride smaller than the lidar packet size");
    if (b->n_slots > kMaxSlots) return fail(OB_INVALID_ARGUMENT, "too many packet slots");
    const size_t F = b->n_frames;
    std::vector<CallLut> frame_luts(b->frame_luts ? F : 0);
    for (size_t f = 0; f < frame_luts.size(); ++f) {
        if (!b->frame_luts[f]) return fail(OB_INVALID_ARGUMENT, "null per-frame lut");
        if ((rs = take_lut(c, b->frame_luts[f], &frame_luts[f])) != OB_OK) return rs;
    }
    if ((rs = check_fused(c, lut || b->frame_luts, b->xyz, b->range_destaggered)) != OB_OK) return rs;

    Staging stg(stream_handle(s));
    auto span = [&](size_t stride, size_t last) { return (F - 1) * stride + last; };
    const uint8_t* dpk =
        stg.in(b->packets, span(b->packets_frame_stride, (b->n_slots - 1) * b->packet_stride + L.packet_size));
    if (cudaError_t e = stg.error()) return fail_cuda(e, "stage packets");
    void* dout[kOuts] = {};       // frame 0's outputs as the kernel writes them ...
    size_t dstride[kOuts] = {};   // ... and the bytes from one frame's to the next's there
    for (int k = 0; k < kOuts; ++k) {
        void* user = io_out(L, *b, k);
        if (!user) continue;
        const size_t fs = batch_stride(*b, k), block = out_bytes(L, c.dtype, k);
        if (F > 1 && fs > block) {
            // a host output with gaps between its frames is decoded into dense scratch and copied back block by
            // block: the gaps (padding, or the frames of another output that shares the allocation) keep the
            // caller's bytes
            dout[k] = stg.out_rows(user, block, fs, F);
            dstride[k] = dout[k] == user ? fs : block;
        } else {
            dout[k] = stg.out(user, span(fs, block));
            dstride[k] = fs;
        }
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage outputs");
    }
    const bool bulk_ok = al16(dpk) && b->packet_stride % 16 == 0 && L.packet_size % 16 == 0 &&
                         b->packets_frame_stride % 16 == 0;
    std::vector<DecodeFrame> hf(F);
    for (size_t f = 0; f < F; ++f) {
        DecodeFrame& d = hf[f];
        std::memset(&d, 0, sizeof(d));
        d.packets = dpk + f * b->packets_frame_stride;
        d.packet_stride = b->packet_stride;
        d.n_slots = static_cast<uint32_t>(b->n_slots);
        for (int k = 0; k < kOuts; ++k)
            if (dout[k]) set_out(d, k, static_cast<uint8_t*>(dout[k]) + f * dstride[k]);
        finish_frame(c, d, bulk_ok, frame_luts.empty() ? nullptr : &frame_luts[f]);
    }
    // the frames' XYZ pointers show a stride that breaks alignment only when there are two of them
    const size_t xs0 = dstride[kOutReturns], xs1 = dstride[kOutReturns + 2];
    if (c.any_xyz && (xs0 | xs1) % 16) c.vec_ok = false;
    // the XYZ outputs as one strided batch: only when both returns are written with one frame stride
    const bool one_xyz_stride = !dout[kOutReturns] || !dout[kOutReturns + 2] || xs0 == xs1;
    const void* xyz_base[OB_MAX_RETURNS] = {hf[0].xyz[0], hf[0].xyz[1]};
    return run_table(c, s, hf, stg, one_xyz_stride ? xyz_base : nullptr, xs0);
}


// ---------------------------------------------------------------------------------------------
// decode job
// ---------------------------------------------------------------------------------------------
struct ob_decode_job {
    const ob_decoder* dec;
    ob_stream* s;
    cudaStream_t st;
    int device;
    size_t stride;        // bytes per packet slot on the device (multiple of 16)
    DeviceBlock pk;       // packet slots
    size_t cap_slots{0};
    size_t up_slots{0};   // highest uploaded slot + 1
    DeviceBlock out;      // output slab (fields, headers, xyz, destaggered ranges)
    DeviceBlock colsrc;   // int32 x W
    PinnedBlock h_colsrc;
    DeviceBlock frame;    // one DecodeFrame
    PinnedBlock h_frame;
    Event ev_up, ev_done;
    bool up_pending{false}, busy{false};
};

static cudaError_t job_reserve(ob_decode_job* j, size_t slots) {
    if (slots <= j->cap_slots) return cudaSuccess;
    const size_t cap = std::max(slots, j->cap_slots ? j->cap_slots * 2 : static_cast<size_t>(16));
    DeviceBlock p;
    cudaError_t e = p.alloc(cap * j->stride + 16);
    if (e != cudaSuccess) return e;
    if (j->pk.get()) {  // rare: more packets than the frame was sized for (duplicates, retransmits)
        e = cudaStreamSynchronize(j->st);
        if (e == cudaSuccess && j->up_slots)
            e = cudaMemcpy(p.get(), j->pk.get(), j->up_slots * j->stride, cudaMemcpyDeviceToDevice);
        if (e != cudaSuccess) return e;
    }
    j->pk = std::move(p);
    j->cap_slots = cap;
    return cudaSuccess;
}

ob_status ob_decode_job_create(const ob_decoder* dec, size_t reserve_slots, ob_stream* s,
                               ob_decode_job** out) {
    if (!dec || !s || !out) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const int device = dec->device;
    ob_status rs = same_device(dec, s);
    if (rs == OB_OK) rs = require_device(device);
    if (rs != OB_OK) return rs;
    std::unique_ptr<ob_decode_job> j(new ob_decode_job);
    j->dec = dec;
    j->s = s;
    j->st = stream_handle(s);
    j->device = device;
    j->stride = (static_cast<size_t>(dec->L.packet_size) + 15) & ~static_cast<size_t>(15);
    cudaError_t e = j->ev_up.create();
    if (e == cudaSuccess) e = j->ev_done.create();
    if (e == cudaSuccess) e = j->colsrc.alloc(static_cast<size_t>(dec->L.W) * 4);
    if (e == cudaSuccess) e = j->h_colsrc.alloc(static_cast<size_t>(dec->L.W) * 4);
    if (e == cudaSuccess) e = j->frame.alloc(sizeof(DecodeFrame));
    if (e == cudaSuccess) e = j->h_frame.alloc(sizeof(DecodeFrame));
    if (e == cudaSuccess && reserve_slots) e = job_reserve(j.get(), reserve_slots);
    if (e != cudaSuccess) return fail_cuda(e, "decode job allocation");
    *out = j.release();
    return OB_OK;
}

ob_status ob_decode_job_destroy(ob_decode_job* j) {
    if (!j) return OB_OK;
    DeviceScope on(j->device);
    cudaStreamSynchronize(j->st);
    delete j;
    return OB_OK;
}

int ob_decode_job_busy(const ob_decode_job* j) { return j && j->busy ? 1 : 0; }

ob_status ob_decode_job_upload(ob_decode_job* j, const uint8_t* src, size_t src_stride,
                               size_t first_slot, size_t count) {
    if (!j || (count && !src)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (count == 0) return OB_OK;
    const size_t psize = j->dec->L.packet_size;
    if (count > 1 && src_stride < psize)
        return fail(OB_INVALID_ARGUMENT, "packet_stride smaller than the lidar packet size");
    if (first_slot + count > kMaxSlots) return fail(OB_INVALID_ARGUMENT, "too many packet slots");
    ob_status rs = require_device(j->device);
    if (rs != OB_OK) return rs;
    if (j->busy) {  // the previous frame still reads the slots
        rs = ob_decode_job_wait(j);
        if (rs != OB_OK) return rs;
    }
    cudaError_t e = job_reserve(j, first_slot + count);
    if (e != cudaSuccess) return fail_cuda(e, "decode job packet slots");
    uint8_t* dst = j->pk.get<uint8_t>() + first_slot * j->stride;
    if (count == 1 || src_stride == j->stride)
        e = cudaMemcpyAsync(dst, src, (count - 1) * j->stride + psize, cudaMemcpyDefault, j->st);
    else
        e = cudaMemcpy2DAsync(dst, j->stride, src, src_stride, psize, count, cudaMemcpyDefault, j->st);
    if (e != cudaSuccess) return fail_cuda(e, "packet upload");
    e = cudaEventRecord(j->ev_up.get(), j->st);
    if (e != cudaSuccess) return fail_cuda(e, "packet upload event");
    j->up_pending = true;
    // an upload at slot 0 begins a new frame: slots of the previous one are no longer valid
    j->up_slots = first_slot == 0 ? count : std::max(j->up_slots, first_slot + count);
    return OB_OK;
}

ob_status ob_decode_job_uploads_done(ob_decode_job* j) {
    if (!j) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (!j->up_pending) return OB_OK;
    cudaError_t e = cudaEventSynchronize(j->ev_up.get());
    j->up_pending = false;
    if (e != cudaSuccess) return fail_cuda(e, "packet upload");
    return OB_OK;
}

ob_status ob_decode_job_wait(ob_decode_job* j) {
    if (!j) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (!j->busy) return OB_OK;
    cudaError_t e = cudaEventSynchronize(j->ev_done.get());
    j->busy = false;
    j->up_pending = false;
    if (e != cudaSuccess) return fail_cuda(e, "decode job");
    return OB_OK;
}

ob_status ob_decode_job_submit(ob_decode_job* j, const ob_decode_io* io, const ob_lut* lut,
                               const int32_t* shifts, size_t n_shifts) {
    if (!j || !io) return fail(OB_INVALID_ARGUMENT, "null pointer");
    const DecodeLayout& L = j->dec->L;
    // the frame's own LUT replaces the call-level one for the whole one-frame launch; the two share one dtype
    DecodeCall c;
    ob_status rs = begin_call(c, j->dec, j->s, io->lut ? io->lut : lut, shifts, n_shifts);
    if (rs != OB_OK) return rs;
    if (io->n_slots > j->up_slots) return fail(OB_INVALID_ARGUMENT, "n_slots exceeds the uploaded packet slots");
    if (io->lut && lut && lut_view(lut).dtype != c.dtype)
        return fail(OB_INVALID_ARGUMENT, "per-frame lut dtype differs from the call-level lut");
    if ((rs = check_fused(c, io->lut || lut, io->xyz, io->range_destaggered)) != OB_OK) return rs;
    if (j->busy) {  // the previous submission still owns h_frame / h_colsrc / the slab
        rs = ob_decode_job_wait(j);
        if (rs != OB_OK) return rs;
    }

    // ---- outputs: device pointers in place, host pointers through the slab + D2H ----
    struct Out {
        void* user;
        size_t bytes;
        int k;
        bool host;
        size_t off;
    };
    Out outs[kOuts];
    size_t n_out = 0;
    for (int k = 0; k < kOuts; ++k)
        if (void* user = io_out(L, *io, k)) outs[n_out++] = Out{user, out_bytes(L, c.dtype, k), k, false, 0};
    // host outputs take slab space in ADDRESS order; buffers that are adjacent in host memory
    // (HostBuffer::carve) stay adjacent in the slab, so their D2H is one copy
    size_t order[kOuts];
    size_t n_host = 0;
    for (size_t i = 0; i < n_out; ++i) {
        outs[i].host = !is_device_ptr(outs[i].user);
        if (outs[i].host) order[n_host++] = i;
    }
    std::sort(order, order + n_host, [&](size_t a, size_t b) {
        return reinterpret_cast<uintptr_t>(outs[a].user) < reinterpret_cast<uintptr_t>(outs[b].user);
    });
    size_t need = 0;
    for (size_t k = 0; k < n_host; ++k) {
        Out& o = outs[order[k]];
        const bool adjacent = k > 0 && static_cast<uint8_t*>(outs[order[k - 1]].user) + outs[order[k - 1]].bytes ==
                                           static_cast<uint8_t*>(o.user) &&
                              (need % 16) == 0;
        if (!adjacent) need = (need + 255) & ~static_cast<size_t>(255);
        o.off = need;
        need += o.bytes;
    }
    cudaError_t e = j->out.reserve(need);  // job is idle here
    if (e != cudaSuccess) return fail_cuda(e, "decode job output slab");
    uint8_t* slab = j->out.get<uint8_t>();
    DecodeFrame f;
    std::memset(&f, 0, sizeof(f));
    for (size_t i = 0; i < n_out; ++i) set_out(f, outs[i].k, outs[i].host ? slab + outs[i].off : outs[i].user);
    f.packets = j->pk.get<uint8_t>();
    f.packet_stride = j->stride;
    f.n_slots = static_cast<uint32_t>(io->n_slots);
    if (io->col_src) {
        std::memcpy(j->h_colsrc.get(), io->col_src, static_cast<size_t>(L.W) * 4);
        e = cudaMemcpyAsync(j->colsrc.get(), j->h_colsrc.get(), static_cast<size_t>(L.W) * 4, cudaMemcpyHostToDevice,
                            j->st);
        if (e != cudaSuccess) return fail_cuda(e, "stage column map");
        f.col_src = j->colsrc.get<int32_t>();
    }
    finish_frame(c, f, L.packet_size % 16 == 0, nullptr);  // slots are 16-byte aligned by construction
    *j->h_frame.get<DecodeFrame>() = f;
    e = cudaMemcpyAsync(j->frame.get(), j->h_frame.get(), sizeof(DecodeFrame), cudaMemcpyHostToDevice, j->st);
    if (e != cudaSuccess) return fail_cuda(e, "frame table upload");
    const void* xyz_base[OB_MAX_RETURNS] = {f.xyz[0], f.xyz[1]};  // a one-frame batch
    e = launch(c, j->frame.get<DecodeFrame>(), 1, j->st, xyz_base, out_bytes(L, c.dtype, kOutReturns));  // kOutReturns: XYZ of return 0
    if (e != cudaSuccess) return fail_cuda(e, "decode launch");
    for (size_t k = 0; k < n_host;) {  // one D2H per run of outputs contiguous on both sides
        const Out& first = outs[order[k]];
        size_t bytes = first.bytes, m = k + 1;
        while (m < n_host && outs[order[m]].off == first.off + bytes &&
               static_cast<uint8_t*>(outs[order[m]].user) == static_cast<uint8_t*>(first.user) + bytes) {
            bytes += outs[order[m]].bytes;
            ++m;
        }
        e = cudaMemcpyAsync(first.user, slab + first.off, bytes, cudaMemcpyDeviceToHost, j->st);
        if (e != cudaSuccess) return fail_cuda(e, "decode D2H");
        k = m;
    }
    e = cudaEventRecord(j->ev_done.get(), j->st);
    if (e != cudaSuccess) return fail_cuda(e, "decode job event");
    j->busy = true;
    return OB_OK;
}

ob_status ob_encode_frames(const ob_decoder* dec, const ob_encode_io* frames, size_t n_frames, int with_crc,
                           ob_stream* s) {
    if (!dec || !s || (n_frames && !frames)) return fail(OB_INVALID_ARGUMENT, "null pointer");
    if (n_frames == 0) return OB_OK;
    const DecodeLayout& L = dec->L;
    const int device = dec->device;
    ob_status rs = same_device(dec, s);
    if (rs != OB_OK) return rs;
    if (L.W % L.cpp != 0)
        return fail(OB_INVALID_ARGUMENT, "Mismatch between expected number of packets and PacketFormat.columns_per_packet");
    if (with_crc && (L.packet_size % 4 != 0 || L.packet_size < 8))
        return fail(OB_INVALID_ARGUMENT, "packet size must be a multiple of 4 for the CRC64 footer");
    // The encoder clears and sets each field's mask in place, one thread per pixel.  That gives the reference's
    // result only when no mask reaches into a neighbouring pixel's bytes; which pixel the reference writes
    // last would then decide the overlap, and the encoder does not reproduce that order.
    for (uint32_t k = 0; k < L.n_fields; ++k) {
        const uint64_t m = L.fields[k].mask;
        const uint32_t span = m ? (64u - static_cast<uint32_t>(__builtin_clzll(m)) + 7u) / 8u : 0u;
        if (static_cast<uint64_t>(L.fields[k].offset) + span > L.channel_data_size)
            return fail(OB_INVALID_ARGUMENT, "field mask reaches past the pixel's channel data; cannot encode");
    }
    rs = require_device(device);
    if (rs != OB_OK) return rs;
    cudaStream_t st = stream_handle(s);
    Staging stg(st);
    const size_t n_pk = L.W / L.cpp;
    std::vector<EncodeFrame> hf(n_frames);
    for (size_t i = 0; i < n_frames; ++i) {
        const ob_encode_io& io = frames[i];
        EncodeFrame& f = hf[i];
        std::memset(&f, 0, sizeof(f));
        if (!io.packets) return fail(OB_INVALID_ARGUMENT, "null packet buffer");
        if (io.packet_stride < L.packet_size)
            return fail(OB_INVALID_ARGUMENT, "packet_stride smaller than the lidar packet size");
        if (io.packet_headers && io.packet_header_bytes < L.packet_header_size)
            return fail(OB_INVALID_ARGUMENT, "packet_header_bytes smaller than the packet header");
        for (uint32_t k = 0; k < L.n_fields; ++k)
            if (io.fields[k]) f.fields[k] = stg.in(io.fields[k], out_bytes(L, OB_F32, k));
        if (io.timestamp) f.timestamp = stg.in(io.timestamp, L.W);
        if (io.status) f.status = stg.in(io.status, L.W);
        if (io.packet_headers) {
            f.packet_headers = stg.in(io.packet_headers, n_pk * io.packet_header_bytes);
            f.header_bytes = static_cast<uint32_t>(io.packet_header_bytes);
        }
        // the kernel writes packet_size bytes of every packet_stride; a host buffer with gaps between packets is
        // uploaded first so that its copy back leaves the gaps as the caller had them
        const size_t span = (n_pk - 1) * io.packet_stride + L.packet_size;
        f.packets = io.packet_stride == L.packet_size ? stg.out(io.packets, span) : stg.inout(io.packets, span);
        if (cudaError_t e = stg.error()) return fail_cuda(e, "stage encode buffers");
        f.packet_stride = io.packet_stride;
    }
    const void* fdev = nullptr;
    cudaError_t e = stream_table(s, 1, hf.data(), n_frames * sizeof(EncodeFrame), &fdev);
    if (e != cudaSuccess) return fail_cuda(e, "frame table upload");
    e = launch_encode(L, static_cast<const EncodeFrame*>(fdev), static_cast<uint32_t>(n_frames), with_crc != 0, device, st);
    if (e != cudaSuccess) return fail_cuda(e, "encode launch");
    e = stg.flush();
    if (e != cudaSuccess) return fail_cuda(e, "encode D2H");
    return OB_OK;
}

int ob_pointer_kind(const void* p) {
    if (!p) return 0;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    if (at.type == cudaMemoryTypeHost) return 1;
    if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) return 2;
    return 0;
}

int ob_pointer_host_readable(const void* p) {
    if (!p) return 0;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();
        return 1;
    }
    return at.type == cudaMemoryTypeDevice ? 0 : 1;
}

}  // extern "C"
