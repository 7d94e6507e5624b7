/*
 * ouster_oracle.h -- CPU oracle for the scan->pointcloud hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This is a plain-C restatement of the reference's
 * CPU algorithm for packet decode -> FrameBatcher -> destagger -> cartesian,
 * used as the parity checker.  Only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py may load it.  Nothing in
 * the product path (ouster-sdk_b200/) may include, link or call this file.
 *
 * Parity status: PINNED.  The restatement is checked (tests/test_oracle_*.py)
 * against the reference's own golden data: md5 field digests of 5 pcaps
 * (tests/pcaps/\*_digest.json), the 64-bit snapshot hashes of
 * tests/frame_batcher_test.cpp:548-611, the python doc-formula XYZ and the
 * np.roll destagger of python/src/ouster/sdk/examples/reference.py (imported
 * unmodified when generating tests/golden).
 *
 * All file:line citations are relative to /root/reference (ouster-sdk 1.0.1).
 */
#ifndef OUSTER_ORACLE_H
#define OUSTER_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ChanFieldType tags -- ouster_core/include/ouster/core/chanfield.h:111-128 */
enum {
    ORC_VOID = 0, ORC_UINT8 = 1, ORC_UINT16 = 2, ORC_UINT32 = 3, ORC_UINT64 = 4,
    ORC_INT8 = 5, ORC_INT16 = 6, ORC_INT32 = 7, ORC_INT64 = 8,
    ORC_FLOAT32 = 9, ORC_FLOAT64 = 10, ORC_CHAR = 11, ORC_FLOAT16 = 12
};

/* UDPProfileLidar -- ouster_core/include/ouster/core/data_format.h:27-72 */
enum {
    ORC_PROFILE_UNKNOWN = 0,
    ORC_PROFILE_LEGACY = 1,
    ORC_PROFILE_RNG19_RFL8_SIG16_NIR16_DUAL = 2,
    ORC_PROFILE_RNG19_RFL8_SIG16_NIR16 = 3,
    ORC_PROFILE_RNG15_RFL8_NIR8 = 4,
    ORC_PROFILE_FIVE_WORD_PIXEL = 5,
    ORC_PROFILE_FUSA_RNG15_RFL8_NIR8_DUAL = 6,
    ORC_PROFILE_RNG15_RFL8_NIR8_DUAL = 7,
    ORC_PROFILE_RNG15_RFL8_NIR8_ZONE16 = 8,
    ORC_PROFILE_RNG19_RFL8_SIG16_NIR16_ZONE16 = 9,
    ORC_PROFILE_RNG15_RFL8_WIN8 = 10,
    ORC_PROFILE_RNG19_RFL8_SIG16_ZONE16_DUAL = 11,
    ORC_PROFILE_RNG19_RFL8_SIG16_NIR16_RGB16 = 12,
    ORC_PROFILE_RNG19_RFL8_SIG16_NIR16_RGB16_DUAL = 13
};

/* HeaderType -- data_format.h:91-97 */
enum { ORC_HEADER_STANDARD = 0, ORC_HEADER_FUSA = 1 };

/* FieldDecodeInfo -- ouster_core/include/ouster/core/field_decode_info.h:24-79 */
typedef struct orc_field_info {
    int ty_tag;
    size_t offset;
    uint64_t mask;
    int shift;
    int num_elements;
} orc_field_info;

#define ORC_MAX_FIELDS 24
#define ORC_NAME_LEN 24

typedef struct orc_named_field {
    char name[ORC_NAME_LEN];
    orc_field_info info;
} orc_named_field;

/* PacketFormat geometry + header decode infos -- ouster_core/src/parsing.cpp:386-598 */
typedef struct orc_packet_format {
    int profile;
    int header_type;
    uint32_t pixels_per_column;
    uint32_t columns_per_packet;
    uint32_t columns_per_frame;
    size_t packet_header_size, col_header_size, channel_data_size;
    size_t col_footer_size, packet_footer_size, col_size, lidar_packet_size;
    uint32_t max_frame_id;
    int n_fields; /* sorted by name: std::map iteration order, parsing.cpp:406,475 */
    orc_named_field fields[ORC_MAX_FIELDS];
    orc_field_info packet_type_info, frame_id_info, init_id_info, prod_sn_info;
    orc_field_info alert_flags_info, countdown_thermal_shutdown_info;
    orc_field_info countdown_shot_limiting_info, thermal_shutdown_info, shot_limiting_info;
    orc_field_info col_status_info, col_timestamp_info, col_measurement_id_info;
} orc_packet_format;

/* field of an oracle frame (row-major h x w of elem_size bytes) */
typedef struct orc_frame_field {
    char name[ORC_NAME_LEN];
    int ty_tag;
    size_t elem_size;
    uint8_t* data; /* h*w*elem_size, calloc'd */
} orc_frame_field;

/* LidarFrame stand-in -- lidar_frame.h:124-821 (only what the batcher touches) */
typedef struct orc_frame {
    size_t w, h, n_packets;
    int64_t frame_id;
    uint64_t frame_status;
    uint8_t shutdown_countdown, shot_limiting_countdown;
    int n_fields;
    orc_frame_field fields[ORC_MAX_FIELDS];
    uint64_t* timestamp;        /* w */
    uint16_t* measurement_id;   /* w */
    uint32_t* status;           /* w */
    uint64_t* packet_timestamp; /* w / columns_per_packet */
    uint8_t* alert_flags;       /* w / columns_per_packet */
} orc_frame;

typedef struct orc_batcher orc_batcher; /* FrameBatcher -- lidar_frame.cpp:1248-1959 */

/* ---- field_info / FieldDecodeInfo ---- */
int orc_field_info_make(size_t bit_start, size_t bit_size, size_t upshift, size_t max_length,
                        size_t num_elements, orc_field_info* out);
uint64_t orc_field_get(const orc_field_info* fi, const uint8_t* buffer);
void orc_field_set(const orc_field_info* fi, uint8_t* buffer, uint64_t value);
uint64_t orc_value_mask(const orc_field_info* fi);
size_t orc_type_size(int ty_tag);

/* ---- PacketFormat ---- */
int orc_packet_format_init(orc_packet_format* pf, int profile, int header_type,
                           uint32_t pixels_per_column, uint32_t columns_per_packet,
                           uint32_t columns_per_frame);
/* replace the profile's field table (add_custom_profile analogue, profile_extension.cpp:86-185) */
int orc_packet_format_set_fields(orc_packet_format* pf, const orc_named_field* fields, int n,
                                 size_t channel_data_size);
const orc_field_info* orc_pf_field(const orc_packet_format* pf, const char* name);
int orc_block_parsable(const orc_packet_format* pf);
int orc_frame_id_difference(const orc_packet_format* pf, uint32_t current, uint32_t other);
uint64_t orc_crc64(const uint8_t* buf, size_t len);
/* default frame field dtype for a profile field, 0 (VOID) if the field is not in the default set */
int orc_default_field_type(int profile, const char* name);

/* whole-packet field decode, both variants (parsing.cpp:628-675); dst is h x cols row-major */
int orc_block_field(const orc_packet_format* pf, const char* name, size_t elem_size, void* dst,
                    int cols, const uint8_t* lidar_buf, int block_dim);
int orc_col_field(const orc_packet_format* pf, const char* name, size_t elem_size,
                  const uint8_t* col_buf, void* dst, int dst_stride);

/* ---- frame ---- */
orc_frame* orc_frame_create(const orc_packet_format* pf, int with_window);
int orc_frame_add_field(orc_frame* f, const char* name, int ty_tag);
orc_frame_field* orc_frame_field_by_name(orc_frame* f, const char* name);
void orc_frame_destroy(orc_frame* f);

/* ---- batcher ---- */
orc_batcher* orc_batcher_create(const orc_packet_format* pf, uint32_t init_id,
                                uint32_t column_window_first, uint32_t column_window_second);
void orc_batcher_destroy(orc_batcher* b);
/* returns 1 when frame complete, 0 otherwise, <0 on error (-1 invalid_argument, -2 runtime_error) */
int orc_batcher_batch(orc_batcher* b, const uint8_t* buf, size_t len, uint64_t host_timestamp,
                      orc_frame* frame);
void orc_batcher_reset(orc_batcher* b);
size_t orc_batcher_batched_packets(const orc_batcher* b);
size_t orc_batcher_dropped_packets(const orc_batcher* b);
int orc_batcher_set_max_cache_size(orc_batcher* b, size_t n);
void orc_batcher_force_col_path(orc_batcher* b, int on); /* test hook: always parse_by_col */

/* ---- frame_to_packets (lidar part) -- impl/lidar_frame_impl.h:435-531 ---- */
/* writes up to n_packets packets of pf->lidar_packet_size into out; host timestamps into ts_out.
 * returns number of packets emitted */
int orc_frame_to_packets(const orc_frame* f, const orc_packet_format* pf, uint32_t init_id,
                         uint64_t prod_sn, uint8_t* out, uint64_t* ts_out);

/* ---- destagger -- impl/lidar_frame_impl.h:733-811 ---- */
int orc_destagger(size_t elem_size, size_t k, const void* img, const int* shifts, size_t n_shifts,
                  size_t h, size_t w, int inverse, void* out);

/* ---- cartesian -- impl/cartesian.h:36-66 ---- */
void orc_cartesian_f64(double* pts, const uint32_t* rng, const double* dir, const double* ofs,
                       size_t n);
void orc_cartesian_f32(float* pts, const uint32_t* rng, const float* dir, const float* ofs,
                       size_t n);
/* OpenMP variants (the reference's opt-in OUSTER_OMP mode, impl/cartesian.h:15-23,50-52) */
void orc_cartesian_f64_omp(double* pts, const uint32_t* rng, const double* dir, const double* ofs,
                           size_t n);
void orc_cartesian_f32_omp(float* pts, const uint32_t* rng, const float* dir, const float* ofs,
                           size_t n);

/* ---- make_xyz_lut -- ouster_core/src/xyzlut.cpp:11-89 ---- */
int orc_make_xyz_lut(size_t w, size_t h, double range_unit, const double* beam_to_lidar /*4x4 rm*/,
                     const double* transform /*4x4 rm*/, const double* az_deg, size_t n_az,
                     const double* alt_deg, size_t n_alt, double* direction, double* offset);

/* ---- dewarp / transform -- ouster_core/include/ouster/core/pose_util.h:37-59, 118-131 ----
 * out[i*W + w] = R_w * p[i*W + w] + t_w, poses = W x 16 (row-major 4x4 each); n = H*W points.
 * The 3-term dot products are summed as x0 + (x1 + x2) (Eigen's redux_novec_unroller split for
 * length 3); the reference's own test only pins this to rtol 1e-5 (python/tests/test_pose_util.py:334-360). */
void orc_dewarp_f64(double* out, const double* pts, const double* poses, size_t n, size_t w);
void orc_dewarp_f32(float* out, const float* pts, const float* poses, size_t n, size_t w);

/* dewarp<T>(LidarFrame, XYZLutT<T>, min_range, max_range) -- pose_util.h:456-485 ->
 * impl::dewarp_impl, impl/dewarp_impl.h:22-76.  out holds up to h*w points; col_idx / ts_out may be
 * NULL.  poses = LidarFrame::body_to_world (w x 16 doubles).  Returns the number of points. */
size_t orc_dewarp_frame_f64(double* out, uint32_t* col_idx, uint64_t* ts_out, const uint32_t* range,
                            const double* dir, const double* off, const double* poses,
                            const uint32_t* status, const uint64_t* timestamps, size_t h, size_t w,
                            double min_range, double max_range);
size_t orc_dewarp_frame_f32(float* out, uint32_t* col_idx, uint64_t* ts_out, const uint32_t* range,
                            const float* dir, const float* off, const double* poses,
                            const uint32_t* status, const uint64_t* timestamps, size_t h, size_t w,
                            double min_range, double max_range);

/* ---- surface normals on destaggered XYZ -- ouster_algorithm/src/normals.cpp:32-483 (orc_normals.c) ----
 * xyz: h*w x 3 doubles (destaggered), range: h x w, origins: w x 3 (per-column sensor origin) or NULL.
 * orc_normals: single return when xyz2/range2 are NULL (normals.cpp:411-430), else both returns with
 * the first return's vertical subtent passed to both passes (:432-483); a pass given a subtent <= 0
 * derives its own, so the second return's pass uses the subtent of (xyz2, range2) when the first
 * return's is 0.  subtent_override <= 0: derive it from the first return.
 * returns 0, -1 "normals: target_distance_m must be positive", -2 "normals: min_angle_of_incidence_rad
 * must be positive". */
double orc_normals_vertical_subtent(const double* xyz, const uint32_t* range, const double* origins,
                                    size_t h, size_t w);
int orc_normals_compute(const double* xyz, const uint32_t* range, const double* xyz2,
                        const uint32_t* range2, size_t h, size_t w, const double* origins,
                        double* normals, size_t search, double min_aoi_rad, double target_m,
                        double subtent_override);
int orc_normals(const double* xyz, const uint32_t* range, const double* xyz2, const uint32_t* range2,
                size_t h, size_t w, const double* origins, size_t search, double min_aoi_rad,
                double target_m, double subtent_override, double* n1, double* n2);

/* std::hash-combine snapshot of a field, tests/frame_batcher_test.cpp:595-606 */
uint64_t orc_snapshot_hash(const void* data, size_t n, size_t elem_size);

#ifdef __cplusplus
}
#endif
#endif
