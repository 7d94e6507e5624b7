/*
 * ouster_b200_host.h -- C ABI over the host-side mirror of the reference's C++ classes
 * (SensorInfo/PacketFormat, LidarFrame/LidarScan, FrameBatcher/ScanBatcher).  It exists so that
 * non-C++ callers (the Python tests, bench.py, other FFIs) can drive the same objects a C++ caller
 * gets from include/ouster/core/ (reference headers: lidar_frame.h, types.h, xyzlut.h).
 * Status/err conventions are those of ouster_b200.h (ob_last_error()).
 */
#ifndef OUSTER_B200_HOST_H
#define OUSTER_B200_HOST_H

#include "ouster_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct obh_sensor obh_sensor;   /* SensorInfo + its PacketFormat */
typedef struct obh_frame obh_frame;     /* LidarFrame (LidarScan) */
typedef struct obh_batcher obh_batcher; /* FrameBatcher (ScanBatcher) */

/* CUDA device used by the calling thread's host-mirror objects (FrameBatcher, XYZLut, destagger);
 * default 0 or env OUSTER_B200_DEVICE (b200::set_device) */
ob_status obh_set_device(int device);
int obh_get_device(void);

/* ---- SensorInfo / PacketFormat (types.h:109-1116, sensor_info.h:171-244) ---- */
ob_status obh_sensor_create(const char* udp_profile_lidar, int header_type_fusa,
                            uint32_t pixels_per_column, uint32_t columns_per_frame,
                            uint32_t columns_per_packet, const int32_t* pixel_shift_by_row,
                            uint32_t init_id, uint64_t serial_no, const char* fw_rev,
                            uint32_t column_window_first, uint32_t column_window_second,
                            obh_sensor** out);
ob_status obh_sensor_set_intrinsics(obh_sensor* s, const double* azimuth_deg, size_t n_az,
                                    const double* altitude_deg, size_t n_alt,
                                    const double* beam_to_lidar16, const double* lidar_to_sensor16,
                                    const double* sensor_to_body16 /* nullable */);
/* add_custom_profile analogue: replaces the channel field table of this sensor's packet format */
ob_status obh_sensor_set_custom_fields(obh_sensor* s, size_t n, const char* const* names,
                                       const int32_t* ty_tags, const uint64_t* offsets,
                                       const uint64_t* masks, const int32_t* shifts,
                                       size_t channel_data_size);
ob_status obh_sensor_layout(const obh_sensor* s, ob_packet_layout* out);
size_t obh_sensor_n_fields(const obh_sensor* s);
/* i-th profile field in PacketFormat iteration (std::map) order */
ob_status obh_sensor_field(const obh_sensor* s, size_t i, char* name, size_t name_cap,
                           int32_t* ty_tag, uint64_t* offset, uint64_t* mask, int32_t* shift,
                           int32_t* num_elements, uint64_t* value_mask);
int obh_sensor_block_parsable(const obh_sensor* s);
int obh_sensor_frame_id_difference(const obh_sensor* s, uint32_t current, uint32_t other);
uint32_t obh_sensor_packet_frame_id(const obh_sensor* s, const uint8_t* packet);
uint32_t obh_sensor_packet_init_id(const obh_sensor* s, const uint8_t* packet);
uint64_t obh_sensor_packet_prod_sn(const obh_sensor* s, const uint8_t* packet);
uint64_t obh_sensor_calculate_crc(const obh_sensor* s, const uint8_t* packet, size_t size);
ob_status obh_sensor_destroy(obh_sensor* s);

/* ---- LidarFrame ---- */
/* default field set of the sensor's profile and firmware (get_field_types(info)) */
ob_status obh_frame_create(const obh_sensor* s, obh_frame** out);
ob_status obh_frame_add_field(obh_frame* f, const char* name, int32_t ty_tag, size_t extra_dim);
/* LidarFrame::add_field(name, type, extra_dims, field_class) (lidar_frame.h): field_class is a FieldClass
 * (1 PIXEL_FIELD, 2 COLUMN_FIELD, 3 PACKET_FIELD, 4 FRAME_FIELD); extra_dim > 1 adds one trailing dimension */
ob_status obh_frame_add_field_class(obh_frame* f, const char* name, int32_t ty_tag, size_t extra_dim,
                                    int32_t field_class);
/* LidarFrame::del_field(name): the field is dropped (std::invalid_argument when the frame has no such field) */
ob_status obh_frame_del_field(obh_frame* f, const char* name);
/* class and shape of a field: *ndim dimensions into shape[0..min(*ndim, 8)) */
ob_status obh_frame_field_shape(obh_frame* f, const char* name, int32_t* field_class, size_t* ndim, size_t* shape);
size_t obh_frame_n_fields(const obh_frame* f);
ob_status obh_frame_field_at(obh_frame* f, size_t i, char* name, size_t name_cap, int32_t* ty_tag,
                             size_t* elem_bytes /* incl. trailing dims */, void** data);
ob_status obh_frame_field(obh_frame* f, const char* name, int32_t* ty_tag, size_t* elem_bytes,
                          void** data);
ob_status obh_frame_headers(obh_frame* f, uint64_t** timestamp, uint16_t** measurement_id,
                            uint32_t** status, uint64_t** packet_timestamp, uint8_t** alert_flags,
                            size_t* w, size_t* h, size_t* n_packets);
/* LidarFrame::body_to_world (lidar_frame.h:732-736): w x 4 x 4 doubles, identity on construction */
ob_status obh_frame_body_to_world(obh_frame* f, double** poses);
/* get_first_valid_column / get_last_valid_column (lidar_frame.cpp:907-925); returns 0 when no
 * column has status bit 0 set (the C++ functions throw), else 1 */
int obh_frame_valid_columns(const obh_frame* f, int* first, int* last);
int64_t obh_frame_get_frame_id(const obh_frame* f);
void obh_frame_set_frame_id(obh_frame* f, int64_t id);
uint64_t obh_frame_get_status(const obh_frame* f, uint8_t* shutdown_countdown,
                              uint8_t* shot_limiting_countdown);
void obh_frame_set_status(obh_frame* f, uint64_t frame_status, uint8_t shutdown_countdown,
                          uint8_t shot_limiting_countdown);
ob_status obh_frame_destroy(obh_frame* f);

/* frame_to_packets (impl/lidar_frame_impl.h:435-531): out holds up to n_packets packets of
 * packet_size bytes; returns the number emitted through n_out */
ob_status obh_frame_to_packets(const obh_frame* f, const obh_sensor* s, uint32_t init_id,
                               uint64_t prod_sn, uint8_t* out, uint64_t* host_ts, size_t* n_out);
/* the same packets, produced by the GPU encoder (K4, ob_encode_frames); byte-identical */
ob_status obh_frame_to_packets_device(const obh_frame* f, const obh_sensor* s, uint32_t init_id,
                               uint64_t prod_sn, uint8_t* out, uint64_t* host_ts, size_t* n_out);

/* ---- FrameBatcher ---- */
ob_status obh_batcher_create(const obh_sensor* s, obh_batcher** out);
/* FrameBatcher::batch: *complete = 1 when the frame is ready to use */
ob_status obh_batcher_batch(obh_batcher* b, const uint8_t* packet, size_t size,
                            uint64_t host_timestamp, obh_frame* frame, int* complete);
/* burst form: n packets `stride` bytes apart, fed in order; stops after the packet that completes a
 * frame.  *consumed = packets taken, *complete = 1 if that last packet completed the frame. */
ob_status obh_batcher_batch_burst(obh_batcher* b, const uint8_t* packets, size_t n, size_t stride,
                                  size_t size, const uint64_t* host_timestamps, obh_frame* frame,
                                  size_t* consumed, int* complete);
ob_status obh_batcher_flush(obh_batcher* b, obh_frame* frame);
ob_status obh_batcher_reset(obh_batcher* b);
size_t obh_batcher_batched_packets(const obh_batcher* b);
size_t obh_batcher_dropped_packets(const obh_batcher* b);
size_t obh_batcher_gpu_launches(const obh_batcher* b);
ob_status obh_batcher_set_max_cache_size(obh_batcher* b, size_t n);
/* header-only batching: state machine + headers, no pixel decode (no GPU work) */
ob_status obh_batcher_set_headers_only(obh_batcher* b, int on);
/* fused XYZ (+ destaggered range when shifts != NULL) produced by the decode launch */
ob_status obh_batcher_set_fused(obh_batcher* b, ob_lut* lut /* borrowed; NULL detaches */,
                                const int32_t* pixel_shift_by_row, size_t n_shifts);
ob_status obh_batcher_fused_outputs(obh_batcher* b, int ret, void** xyz, size_t* xyz_bytes,
                                    uint32_t** range_destaggered);
/* FrameBatcher::set_device_outputs: decode the named fields (and, with a fused cloud, XYZ / destaggered
 * range per return; arrays of 2 pointers or NULL) straight into DEVICE buffers, so that the results stay
 * in HBM for the next GPU consumer.  n_fields == 0 and NULL arrays detach.  Headers still go to the frame.
 * error: "device outputs must be device memory" */
ob_status obh_batcher_set_device_outputs(obh_batcher* b, size_t n_fields, const char* const* names,
                                         void* const* field_ptrs, void* const* xyz,
                                         uint32_t* const* range_destaggered);
/* FrameBatcher::set_pipeline_depth / wait (frame == NULL: wait_all) -- see lidar_frame.h */
ob_status obh_batcher_set_pipeline_depth(obh_batcher* b, size_t n);
ob_status obh_batcher_wait(obh_batcher* b, obh_frame* frame);
ob_status obh_batcher_destroy(obh_batcher* b);

/* ---- PcapLidarSource (include/ouster/core/pcap_source.h): capture file -> page-locked ring of lidar packets ----
 * replaces, for this path, the read loop of ouster_pcap/src/pcap_packet_source.cpp (classic pcap, Ethernet/IPv4/UDP,
 * unfragmented).  A burst (pointer, stride, capture timestamps in ns) feeds obh_batcher_batch_burst /
 * obh_pipeline_push_burst in place.  errors: "Failed to open pcap file", "Unsupported pcap format". */
typedef struct obh_pcap obh_pcap;
ob_status obh_pcap_open(const char* path, size_t lidar_packet_size, uint16_t dst_port, size_t ring_packets,
                        obh_pcap** out);
ob_status obh_pcap_next_burst(obh_pcap* p, size_t max_packets, const uint8_t** packets, size_t* stride,
                              const uint64_t** timestamps_ns, size_t* n);
size_t obh_pcap_packets_read(const obh_pcap* p);
size_t obh_pcap_skipped(const obh_pcap* p);
ob_status obh_pcap_close(obh_pcap* p);

/* ---- FramePipeline (include/ouster/core/frame_pipeline.h): ring of frames, `depth` in flight ---- */
typedef struct obh_pipeline obh_pipeline;
typedef struct obh_slot {
    obh_frame* frame;  /* borrowed view of the finished slot's LidarFrame; NULL = no frame finished.
                          Valid until the next slot is returned. */
    void* xyz[2];      /* fused cloud of the slot (NULL when not requested) */
    uint32_t* range_destaggered[2];
    size_t xyz_bytes;
} obh_slot;
ob_status obh_pipeline_create(const obh_sensor* s, size_t depth, ob_lut* lut /* nullable, borrowed */,
                              const int32_t* pixel_shift_by_row, size_t n_shifts, obh_pipeline** out);
ob_status obh_pipeline_push_burst(obh_pipeline* p, const uint8_t* packets, size_t n, size_t stride,
                                  size_t size, const uint64_t* host_timestamps, size_t* consumed,
                                  obh_slot* done);
ob_status obh_pipeline_drain(obh_pipeline* p, obh_slot* done);
/* FrameBatcher::Stats of the pipeline's batcher: ns_burst, ns_upload_wait, ns_submit, ns_wait, frames */
ob_status obh_pipeline_stats(const obh_pipeline* p, uint64_t* out5);
size_t obh_pipeline_in_flight(const obh_pipeline* p);
size_t obh_pipeline_gpu_launches(const obh_pipeline* p);
size_t obh_pipeline_dropped_packets(const obh_pipeline* p);
ob_status obh_pipeline_destroy(obh_pipeline* p);

#ifdef __cplusplus
}
#endif
#endif
