// host_c_api.cpp -- extern "C" wrappers over the C++ host mirror (include/ouster_b200_host.h).
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>

#include "ouster/core/frame_pipeline.h"
#include "ouster/core/pcap_source.h"
#include "ouster/core/lidar_frame.h"
#include "ouster/core/xyzlut.h"
#include "ouster_b200_host.h"

using namespace ouster::sdk::core;

namespace ob {
ob_status fail(ob_status st, const std::string& msg);  // ob_api.cu
}

struct obh_sensor {
    std::shared_ptr<SensorInfo> info;
    std::unique_ptr<PacketFormat> pf;
    bool custom{false};
};
struct obh_frame {
    LidarFrame own;              // storage of frames created through obh_frame_create
    LidarFrame* borrowed{nullptr};  // pipeline slots expose their frames without owning them
    LidarFrame& ref() { return borrowed ? *borrowed : own; }
    const LidarFrame& ref() const { return borrowed ? *borrowed : own; }
};
struct obh_batcher {
    std::unique_ptr<FrameBatcher> b;
    FusedCloud fused;
    bool fused_on{false};
};

namespace {
template <typename F>
ob_status guard(F&& fn) {
    try {
        fn();
        return OB_OK;
    } catch (const std::invalid_argument& e) {
        return ob::fail(OB_INVALID_ARGUMENT, e.what());
    } catch (const std::out_of_range& e) {
        return ob::fail(OB_INVALID_ARGUMENT, e.what());
    } catch (const std::exception& e) {
        return ob::fail(OB_RUNTIME_ERROR, e.what());
    }
}
mat4d mat_from(const double* v) {
    mat4d m;
    for (int i = 0; i < 16; ++i) m.m[i] = v[i];
    return m;
}
void copy_name(const std::string& s, char* out, size_t cap) {
    if (!out || cap == 0) return;
    std::strncpy(out, s.c_str(), cap - 1);
    out[cap - 1] = 0;
}
size_t elem_bytes_of(const Field& f) {
    size_t e = f.element_size();
    for (size_t d = 2; d < f.shape().size(); ++d) e *= f.shape()[d];
    return e;
}
}  // namespace

extern "C" {

ob_status obh_set_device(int device) {
    return guard([&] {
        if (device < 0) throw std::invalid_argument("invalid CUDA device index");
        b200::set_device(device);
    });
}
int obh_get_device(void) { return b200::device(); }

ob_status obh_sensor_create(const char* profile, int fusa, uint32_t h, uint32_t w, uint32_t cpp,
                            const int32_t* shifts, uint32_t init_id, uint64_t sn, const char* fw_rev,
                            uint32_t cw_first, uint32_t cw_second, obh_sensor** out) {
    return guard([&] {
        if (!out || !profile) throw std::invalid_argument("null pointer");
        auto info = std::make_shared<SensorInfo>();
        info->format.udp_profile_lidar = udp_profile_lidar_of_string(profile);
        if (info->format.udp_profile_lidar == UDPProfileLidar::UNKNOWN)
            throw std::invalid_argument("Unknown lidar udp profile");
        info->format.header_type = fusa ? HeaderType::FUSA : HeaderType::STANDARD;
        info->format.pixels_per_column = h;
        info->format.columns_per_frame = w;
        info->format.columns_per_packet = cpp;
        info->format.column_window = {static_cast<uint16_t>(cw_first), static_cast<uint16_t>(cw_second)};
        if (shifts) info->format.pixel_shift_by_row.assign(shifts, shifts + h);
        else info->format.pixel_shift_by_row.assign(h, 0);
        info->init_id = init_id;
        info->sn = sn;
        if (fw_rev) info->fw_rev = fw_rev;
        auto s = std::make_unique<obh_sensor>();
        s->pf = std::make_unique<PacketFormat>(info->format);
        s->info = std::move(info);
        *out = s.release();
    });
}

ob_status obh_sensor_set_intrinsics(obh_sensor* s, const double* az, size_t n_az, const double* alt,
                                    size_t n_alt, const double* b2l, const double* l2s,
                                    const double* s2b) {
    return guard([&] {
        if (!s || !az || !alt || !b2l || !l2s) throw std::invalid_argument("null pointer");
        s->info->beam_azimuth_angles.assign(az, az + n_az);
        s->info->beam_altitude_angles.assign(alt, alt + n_alt);
        s->info->beam_to_lidar_transform = mat_from(b2l);
        s->info->lidar_to_sensor_transform = mat_from(l2s);
        s->info->sensor_to_body = s2b ? mat_from(s2b) : mat4d::Identity();
    });
}

ob_status obh_sensor_set_custom_fields(obh_sensor* s, size_t n, const char* const* names,
                                       const int32_t* tags, const uint64_t* offsets,
                                       const uint64_t* masks, const int32_t* shifts, size_t cds) {
    return guard([&] {
        if (!s) throw std::invalid_argument("null pointer");
        std::vector<std::pair<std::string, FieldDecodeInfo>> fields;
        for (size_t i = 0; i < n; ++i) {
            FieldDecodeInfo f;
            f.ty_tag = static_cast<ChanFieldType>(tags[i]);
            f.offset = offsets[i];
            f.mask = masks[i];
            f.shift = shifts[i];
            f.num_elements = 1;
            fields.emplace_back(names[i], f);
        }
        s->pf->set_custom_fields(fields, cds);
        s->custom = true;
    });
}

ob_status obh_sensor_layout(const obh_sensor* s, ob_packet_layout* L) {
    return guard([&] {
        if (!s || !L) throw std::invalid_argument("null pointer");
        const PacketFormat& pf = *s->pf;
        std::memset(L, 0, sizeof(*L));
        L->packet_header_size = static_cast<uint32_t>(pf.packet_header_size);
        L->col_header_size = static_cast<uint32_t>(pf.col_header_size);
        L->channel_data_size = static_cast<uint32_t>(pf.channel_data_size);
        L->col_size = static_cast<uint32_t>(pf.col_size);
        L->packet_size = static_cast<uint32_t>(pf.lidar_packet_size);
        L->columns_per_packet = static_cast<uint32_t>(pf.columns_per_packet);
        L->pixels_per_column = static_cast<uint32_t>(pf.pixels_per_column);
        L->columns_per_frame = s->info->format.columns_per_frame;
        auto conv = [](const FieldDecodeInfo& f) {
            ob_field_desc d{};
            d.offset = static_cast<uint32_t>(f.offset);
            d.elem_size = 8;
            d.mask = f.mask;
            d.shift = f.shift;
            d.range_return = -1;
            return d;
        };
        L->col_timestamp = conv(pf.col_timestamp_info());
        L->col_measurement_id = conv(pf.col_measurement_id_info());
        L->col_status = conv(pf.col_status_info());
    });
}

size_t obh_sensor_n_fields(const obh_sensor* s) {
    return s ? static_cast<size_t>(s->pf->end() - s->pf->begin()) : 0;
}

ob_status obh_sensor_field(const obh_sensor* s, size_t i, char* name, size_t cap, int32_t* tag,
                           uint64_t* offset, uint64_t* mask, int32_t* shift, int32_t* nel,
                           uint64_t* value_mask) {
    return guard([&] {
        if (!s || i >= obh_sensor_n_fields(s)) throw std::invalid_argument("field index out of range");
        const auto& e = *(s->pf->begin() + static_cast<std::ptrdiff_t>(i));
        const FieldDecodeInfo& f = s->pf->field_decode_info(e.first);
        copy_name(e.first, name, cap);
        if (tag) *tag = static_cast<int32_t>(f.ty_tag);
        if (offset) *offset = f.offset;
        if (mask) *mask = f.mask;
        if (shift) *shift = f.shift;
        if (nel) *nel = f.num_elements;
        if (value_mask) *value_mask = s->pf->field_value_mask(e.first);
    });
}

int obh_sensor_block_parsable(const obh_sensor* s) { return s->pf->block_parsable(); }
int obh_sensor_frame_id_difference(const obh_sensor* s, uint32_t cur, uint32_t other) {
    return s->pf->frame_id_difference(cur, other);
}
uint32_t obh_sensor_packet_frame_id(const obh_sensor* s, const uint8_t* p) { return s->pf->frame_id(p); }
uint32_t obh_sensor_packet_init_id(const obh_sensor* s, const uint8_t* p) { return s->pf->init_id(p); }
uint64_t obh_sensor_packet_prod_sn(const obh_sensor* s, const uint8_t* p) { return s->pf->prod_sn(p); }
uint64_t obh_sensor_calculate_crc(const obh_sensor* s, const uint8_t* p, size_t n) {
    return s->pf->calculate_crc(p, n);
}
ob_status obh_sensor_destroy(obh_sensor* s) {
    delete s;
    return OB_OK;
}

// ---- LidarFrame ----
ob_status obh_frame_create(const obh_sensor* s, obh_frame** out) {
    return guard([&] {
        if (!s || !out) throw std::invalid_argument("null pointer");
        auto f = std::make_unique<obh_frame>();
        if (s->custom) {
            // custom profile: the frame carries exactly the custom fields at their decoded types
            LidarFrameFieldTypes ft;
            for (auto it = s->pf->begin(); it != s->pf->end(); ++it)
                ft.emplace_back(it->first, it->second.first);
            f->own = LidarFrame(s->info, ft);
        } else {
            f->own = LidarFrame(s->info);
        }
        *out = f.release();
    });
}

ob_status obh_frame_add_field(obh_frame* f, const char* name, int32_t tag, size_t extra) {
    return guard([&] {
        if (!f || !name) throw std::invalid_argument("null pointer");
        std::vector<size_t> ed;
        if (extra > 1) ed.push_back(extra);
        f->ref().add_field(name, static_cast<ChanFieldType>(tag), ed);
    });
}

ob_status obh_frame_add_field_class(obh_frame* f, const char* name, int32_t tag, size_t extra, int32_t cls) {
    return guard([&] {
        if (!f || !name) throw std::invalid_argument("null pointer");
        if (cls < 1 || cls > 4) throw std::invalid_argument("unknown field class");
        std::vector<size_t> ed;
        if (extra > 1) ed.push_back(extra);
        f->ref().add_field(name, static_cast<ChanFieldType>(tag), ed, static_cast<FieldClass>(cls));
    });
}

ob_status obh_frame_del_field(obh_frame* f, const char* name) {
    return guard([&] {
        if (!f || !name) throw std::invalid_argument("null pointer");
        f->ref().del_field(name);
    });
}

ob_status obh_frame_field_shape(obh_frame* f, const char* name, int32_t* cls, size_t* ndim, size_t* shape) {
    return guard([&] {
        if (!f || !name) throw std::invalid_argument("null pointer");
        const Field& fld = f->ref().field(name);
        if (cls) *cls = static_cast<int32_t>(f->ref().field_type(name).field_class);
        if (ndim) *ndim = fld.shape().size();
        if (shape)
            for (size_t i = 0; i < fld.shape().size() && i < 8; ++i) shape[i] = fld.shape()[i];
    });
}

size_t obh_frame_n_fields(const obh_frame* f) { return f ? f->ref().fields().size() : 0; }

ob_status obh_frame_field_at(obh_frame* f, size_t i, char* name, size_t cap, int32_t* tag,
                             size_t* elem_bytes, void** data) {
    return guard([&] {
        if (!f || i >= f->ref().fields().size()) throw std::invalid_argument("field index out of range");
        auto it = f->ref().fields().begin();
        std::advance(it, static_cast<std::ptrdiff_t>(i));
        copy_name(it->first, name, cap);
        if (tag) *tag = static_cast<int32_t>(it->second.tag());
        if (elem_bytes) *elem_bytes = elem_bytes_of(it->second);
        if (data) *data = it->second.get();
    });
}

ob_status obh_frame_field(obh_frame* f, const char* name, int32_t* tag, size_t* elem_bytes, void** data) {
    return guard([&] {
        if (!f || !name) throw std::invalid_argument("null pointer");
        Field& fld = f->ref().field(name);
        if (tag) *tag = static_cast<int32_t>(fld.tag());
        if (elem_bytes) *elem_bytes = elem_bytes_of(fld);
        if (data) *data = fld.get();
    });
}

ob_status obh_frame_headers(obh_frame* f, uint64_t** ts, uint16_t** mid, uint32_t** st,
                            uint64_t** pts, uint8_t** af, size_t* w, size_t* h, size_t* np) {
    return guard([&] {
        if (!f) throw std::invalid_argument("null pointer");
        LidarFrame& fr = f->ref();
        if (ts) *ts = fr.timestamp().data();
        if (mid) *mid = fr.measurement_id().data();
        if (st) *st = fr.status().data();
        if (pts) *pts = fr.packet_timestamp().data();
        if (af) *af = fr.alert_flags().data();
        if (w) *w = fr.w;
        if (h) *h = fr.h;
        if (np) *np = fr.packet_timestamp().size();
    });
}

ob_status obh_frame_body_to_world(obh_frame* f, double** poses) {
    return guard([&] {
        if (!f || !poses) throw std::invalid_argument("null pointer");
        *poses = f->ref().body_to_world().get<double>();
    });
}

int obh_frame_valid_columns(const obh_frame* f, int* first, int* last) {
    try {
        const int a = f->ref().get_first_valid_column(), b = f->ref().get_last_valid_column();
        if (first) *first = a;
        if (last) *last = b;
        return 1;
    } catch (const std::exception&) {
        return 0;
    }
}

int64_t obh_frame_get_frame_id(const obh_frame* f) { return f->ref().frame_id; }
void obh_frame_set_frame_id(obh_frame* f, int64_t id) { f->ref().frame_id = id; }
uint64_t obh_frame_get_status(const obh_frame* f, uint8_t* sc, uint8_t* slc) {
    if (sc) *sc = f->ref().shutdown_countdown;
    if (slc) *slc = f->ref().shot_limiting_countdown;
    return f->ref().frame_status;
}
void obh_frame_set_status(obh_frame* f, uint64_t st, uint8_t sc, uint8_t slc) {
    f->ref().frame_status = st;
    f->ref().shutdown_countdown = sc;
    f->ref().shot_limiting_countdown = slc;
}
ob_status obh_frame_destroy(obh_frame* f) {
    delete f;
    return OB_OK;
}

ob_status obh_frame_to_packets(const obh_frame* f, const obh_sensor* s, uint32_t init_id,
                               uint64_t prod_sn, uint8_t* out, uint64_t* host_ts, size_t* n_out) {
    return guard([&] {
        if (!f || !s || !out || !n_out) throw std::invalid_argument("null pointer");
        auto packets = impl::frame_to_packets(f->ref(), *s->pf, init_id, prod_sn);
        const size_t psz = s->pf->lidar_packet_size;
        for (size_t i = 0; i < packets.size(); ++i) {
            std::memcpy(out + i * psz, packets[i].buf.data(), psz);
            if (host_ts) host_ts[i] = packets[i].host_timestamp;
        }
        *n_out = packets.size();
    });
}

ob_status obh_frame_to_packets_device(const obh_frame* f, const obh_sensor* s, uint32_t init_id,
                                      uint64_t prod_sn, uint8_t* out, uint64_t* host_ts, size_t* n_out) {
    return guard([&] {
        if (!f || !s || !out || !n_out) throw std::invalid_argument("null pointer");
        auto packets = impl::frame_to_packets_device(f->ref(), *s->pf, init_id, prod_sn);
        const size_t psz = s->pf->lidar_packet_size;
        for (size_t i = 0; i < packets.size(); ++i) {
            std::memcpy(out + i * psz, packets[i].buf.data(), psz);
            if (host_ts) host_ts[i] = packets[i].host_timestamp;
        }
        *n_out = packets.size();
    });
}

// ---- PcapLidarSource ----
struct obh_pcap {
    std::unique_ptr<PcapLidarSource> src;
};
ob_status obh_pcap_open(const char* path, size_t lidar_packet_size, uint16_t dst_port, size_t ring_packets,
                        obh_pcap** out) {
    return guard([&] {
        if (!path || !out) throw std::invalid_argument("null pointer");
        auto p = std::make_unique<obh_pcap>();
        p->src = std::make_unique<PcapLidarSource>(path, lidar_packet_size, dst_port, ring_packets);
        *out = p.release();
    });
}
ob_status obh_pcap_next_burst(obh_pcap* p, size_t max_packets, const uint8_t** packets, size_t* stride,
                              const uint64_t** timestamps_ns, size_t* n) {
    return guard([&] {
        if (!p || !n) throw std::invalid_argument("null pointer");
        *n = p->src->next_burst(max_packets, packets, timestamps_ns);
        if (stride) *stride = p->src->stride();
    });
}
size_t obh_pcap_packets_read(const obh_pcap* p) { return p ? p->src->packets_read() : 0; }
size_t obh_pcap_skipped(const obh_pcap* p) { return p ? p->src->skipped() : 0; }
ob_status obh_pcap_close(obh_pcap* p) {
    delete p;
    return OB_OK;
}

// ---- FrameBatcher ----
ob_status obh_batcher_create(const obh_sensor* s, obh_batcher** out) {
    return guard([&] {
        if (!s || !out) throw std::invalid_argument("null pointer");
        auto b = std::make_unique<obh_batcher>();
        b->b = std::make_unique<FrameBatcher>(s->info);
        if (s->custom) b->b->pf = *s->pf;
        *out = b.release();
    });
}

ob_status obh_batcher_batch(obh_batcher* b, const uint8_t* packet, size_t size, uint64_t ts,
                            obh_frame* frame, int* complete) {
    return guard([&] {
        if (!b || !packet || !frame) throw std::invalid_argument("null pointer");
        const bool done = b->b->batch(packet, size, ts, frame->ref());
        if (complete) *complete = done ? 1 : 0;
    });
}

ob_status obh_batcher_batch_burst(obh_batcher* b, const uint8_t* packets, size_t n, size_t stride,
                                  size_t size, const uint64_t* ts, obh_frame* frame,
                                  size_t* consumed, int* complete) {
    return guard([&] {
        if (!b || !packets || !frame || !ts) throw std::invalid_argument("null pointer");
        bool done = false;
        const size_t used = b->b->batch_burst(packets, n, stride, size, ts, frame->ref(), done);
        if (consumed) *consumed = used;
        if (complete) *complete = done ? 1 : 0;
    });
}

ob_status obh_batcher_flush(obh_batcher* b, obh_frame* frame) {
    return guard([&] { b->b->flush(frame->ref()); });
}
ob_status obh_batcher_reset(obh_batcher* b) {
    return guard([&] { b->b->reset(); });
}
size_t obh_batcher_batched_packets(const obh_batcher* b) { return b->b->batched_packets(); }
size_t obh_batcher_dropped_packets(const obh_batcher* b) { return b->b->dropped_packets(); }
size_t obh_batcher_gpu_launches(const obh_batcher* b) { return b->b->gpu_launches(); }
ob_status obh_batcher_set_max_cache_size(obh_batcher* b, size_t n) {
    return guard([&] { b->b->set_max_cache_size(n); });
}

ob_status obh_batcher_set_headers_only(obh_batcher* b, int on) {
    return guard([&] { b->b->set_headers_only(on != 0); });
}

ob_status obh_batcher_set_fused(obh_batcher* b, ob_lut* lut, const int32_t* shifts, size_t n) {
    return guard([&] {
        if (!b) throw std::invalid_argument("null pointer");
        if (!lut) {
            b->b->set_fused_cloud(nullptr);
            b->fused_on = false;
            return;
        }
        int dtype = OB_F32;
        ob_lut_info(lut, nullptr, nullptr, &dtype, nullptr);
        b->fused.lut = std::shared_ptr<ob_lut>(lut, [](ob_lut*) {});  // borrowed
        b->fused.lut_is_f64 = dtype == OB_F64;
        b->fused.pixel_shift_by_row.clear();
        if (shifts) b->fused.pixel_shift_by_row.assign(shifts, shifts + n);
        b->b->set_fused_cloud(&b->fused);
        b->fused_on = true;
    });
}

ob_status obh_batcher_fused_outputs(obh_batcher* b, int ret, void** xyz, size_t* xyz_bytes,
                                    uint32_t** rd) {
    return guard([&] {
        if (!b || ret < 0 || ret >= 2) throw std::invalid_argument("bad return index");
        if (xyz) *xyz = b->fused.xyz[ret].data();
        if (xyz_bytes) *xyz_bytes = b->fused.xyz[ret].size();
        if (rd)
            *rd = b->fused.range_destaggered[ret].size()
                      ? reinterpret_cast<uint32_t*>(b->fused.range_destaggered[ret].data())
                      : nullptr;
    });
}

ob_status obh_batcher_set_device_outputs(obh_batcher* b, size_t n_fields, const char* const* names,
                                         void* const* field_ptrs, void* const* xyz,
                                         uint32_t* const* range_destaggered) {
    return guard([&] {
        if (!b) throw std::invalid_argument("null pointer");
        if (n_fields == 0 && !xyz && !range_destaggered) {
            b->b->set_device_outputs(nullptr);
            return;
        }
        if (n_fields && (!names || !field_ptrs)) throw std::invalid_argument("null pointer");
        FrameBatcher::DeviceOutputs o;
        for (size_t i = 0; i < n_fields; ++i) {
            if (!names[i]) throw std::invalid_argument("null field name");
            if (field_ptrs[i] && ob_pointer_kind(field_ptrs[i]) != 2)
                throw std::invalid_argument("device outputs must be device memory");
            o.fields.emplace_back(names[i], field_ptrs[i]);
        }
        for (int r = 0; r < 2; ++r) {
            if (xyz) o.xyz[r] = xyz[r];
            if (range_destaggered) o.range_destaggered[r] = range_destaggered[r];
        }
        b->b->set_device_outputs(&o);
    });
}

ob_status obh_batcher_set_pipeline_depth(obh_batcher* b, size_t n) {
    return guard([&] { b->b->set_pipeline_depth(n); });
}
ob_status obh_batcher_wait(obh_batcher* b, obh_frame* frame) {
    return guard([&] {
        if (frame) b->b->wait(frame->ref());
        else b->b->wait_all();
    });
}

ob_status obh_batcher_destroy(obh_batcher* b) {
    delete b;
    return OB_OK;
}

// ---- FramePipeline ----
struct obh_pipeline {
    std::unique_ptr<FramePipeline> p;
    std::vector<std::pair<const FramePipeline::Slot*, std::unique_ptr<obh_frame>>> views;
    obh_frame* view(const FramePipeline::Slot* s) {
        for (auto& v : views)
            if (v.first == s) return v.second.get();
        auto f = std::make_unique<obh_frame>();
        f->borrowed = const_cast<LidarFrame*>(&s->frame);
        views.emplace_back(s, std::move(f));
        return views.back().second.get();
    }
};

static void fill_slot_out(obh_pipeline* p, const FramePipeline::Slot* s, obh_slot* out) {
    std::memset(out, 0, sizeof(*out));
    if (!s) return;
    out->frame = p->view(s);
    for (int r = 0; r < 2; ++r) {
        out->xyz[r] = s->cloud.xyz[r].size() ? const_cast<uint8_t*>(s->cloud.xyz[r].data()) : nullptr;
        out->range_destaggered[r] =
            s->cloud.range_destaggered[r].size()
                ? reinterpret_cast<uint32_t*>(const_cast<uint8_t*>(s->cloud.range_destaggered[r].data()))
                : nullptr;
    }
    out->xyz_bytes = s->cloud.xyz[0].size();
}

ob_status obh_pipeline_create(const obh_sensor* s, size_t depth, ob_lut* lut,
                              const int32_t* shifts, size_t n_shifts, obh_pipeline** out) {
    return guard([&] {
        if (!s || !out) throw std::invalid_argument("null pointer");
        if (s->custom) throw std::invalid_argument("FramePipeline does not support custom profiles yet");
        FusedCloud proto;
        if (lut) {
            int dtype = OB_F32;
            ob_lut_info(lut, nullptr, nullptr, &dtype, nullptr);
            proto.lut = std::shared_ptr<ob_lut>(lut, [](ob_lut*) {});  // borrowed
            proto.lut_is_f64 = dtype == OB_F64;
            if (shifts) proto.pixel_shift_by_row.assign(shifts, shifts + n_shifts);
        }
        auto p = std::make_unique<obh_pipeline>();
        p->p = std::make_unique<FramePipeline>(s->info, depth, lut ? &proto : nullptr);
        *out = p.release();
    });
}

ob_status obh_pipeline_push_burst(obh_pipeline* p, const uint8_t* packets, size_t n, size_t stride,
                                  size_t size, const uint64_t* ts, size_t* consumed, obh_slot* done) {
    return guard([&] {
        if (!p || !packets || !ts || !done) throw std::invalid_argument("null pointer");
        const FramePipeline::Slot* s = nullptr;
        const size_t used = p->p->push_burst(packets, n, stride, size, ts, &s);
        if (consumed) *consumed = used;
        fill_slot_out(p, s, done);
    });
}

ob_status obh_pipeline_drain(obh_pipeline* p, obh_slot* done) {
    return guard([&] {
        if (!p || !done) throw std::invalid_argument("null pointer");
        fill_slot_out(p, p->p->drain(), done);
    });
}

ob_status obh_pipeline_stats(const obh_pipeline* p, uint64_t* out5) {
    return guard([&] {
        if (!p || !out5) throw std::invalid_argument("null pointer");
        const FrameBatcher::Stats& st = p->p->batcher().stats();
        out5[0] = st.ns_burst;
        out5[1] = st.ns_upload_wait;
        out5[2] = st.ns_submit;
        out5[3] = st.ns_wait;
        out5[4] = st.frames;
    });
}
size_t obh_pipeline_in_flight(const obh_pipeline* p) { return p ? p->p->in_flight() : 0; }
size_t obh_pipeline_gpu_launches(const obh_pipeline* p) { return p ? p->p->batcher().gpu_launches() : 0; }
size_t obh_pipeline_dropped_packets(const obh_pipeline* p) { return p ? p->p->batcher().dropped_packets() : 0; }

ob_status obh_pipeline_destroy(obh_pipeline* p) {
    delete p;
    return OB_OK;
}

}  // extern "C"
