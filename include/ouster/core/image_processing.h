// image_processing.h -- AutoExposure, BeamUniformityCorrector and LocalToneMapper
// (mirrors ouster_core/include/ouster/core/image_processing.h).  Same class names, constructors, defaults and
// update() overloads; the work runs on the GPU (ob_image_proc_*, ouster-sdk_b200/csrc/ob_image.cu) and each
// object's state lives in device memory.  Images may be host or device memory: a host image is copied, processed
// and copied back before update() returns.
#pragma once
#include <cstddef>
#include <cstdint>
#include <memory>

#include "ouster/core/b200_runtime.h"
#include "ouster/core/chanfield.h"
#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace core {
namespace image {

/// Dense row-major H x W x 3 view, the role Eigen::TensorMap<rgb_img_t<T>> plays in the reference.  A distinct
/// type, so that update(mono) and update(rgb) resolve as the reference's overloads do.
template <typename T>
class RgbImageRef {
   public:
    RgbImageRef(T* data, size_t h, size_t w) : data_(data), h_(h), w_(w) {}
    T* data() const { return data_; }
    /// dimension(0) = H, dimension(1) = W, dimension(2) = 3
    size_t dimension(int i) const { return i == 0 ? h_ : i == 1 ? w_ : 3; }
    size_t size() const { return h_ * w_ * 3; }

   private:
    T* data_;
    size_t h_, w_;
};

namespace impl {
class ImageProc {
   public:
    ImageProc(int kind, double lo, double hi, int update_every, double damping, double compress, bool color) {
        ob_image_params p{lo, hi, update_every, color ? 1 : 0, damping, compress};
        ob_image_proc* h = nullptr;
        b200::check(ob_image_proc_create(b200::device(), kind, &p, &h));
        h_.reset(h, [](ob_image_proc* q) { ob_image_proc_destroy(q); });
    }
    void run(int layout, int dtype, const void* in, void* out, size_t rows, size_t cols, bool update_state) {
        b200::check(ob_image_proc_update(h_.get(), layout, dtype, in, out, uint32_t(rows), uint32_t(cols),
                                         update_state ? 1 : 0, b200::thread_stream()));
        b200::synchronize();
    }
    ob_image_state state(double* dark_count = nullptr, size_t cap = 0) const {
        ob_image_state s{};
        b200::check(ob_image_proc_state(h_.get(), &s, dark_count, cap, b200::thread_stream()));
        return s;
    }

   private:
    std::shared_ptr<ob_image_proc> h_;
};
}  // namespace impl

/// Adjusts brightness to between 0 and 1 (image_processing.cpp:201-405).
class AutoExposure {
   public:
    AutoExposure() : AutoExposure(0.1, 0.1, 3) {}
    AutoExposure(int update_every) : AutoExposure(0.1, 0.1, update_every) {}
    AutoExposure(double lo_percentile, double hi_percentile, int update_every, double damping = 0.9)
        : p_(OB_IMAGE_AUTO_EXPOSURE, lo_percentile, hi_percentile, update_every, damping, 0.0, false) {}

    void update(ArrayRef<float> image, bool update_state = true) {
        p_.run(OB_IMAGE_MONO, OB_F32, nullptr, image.data(), image.rows(), image.cols(), update_state);
    }
    void update(ArrayRef<double> image, bool update_state = true) {
        p_.run(OB_IMAGE_MONO, OB_F64, nullptr, image.data(), image.rows(), image.cols(), update_state);
    }
    void update(RgbImageRef<float> image, bool update_state = true) {
        p_.run(OB_IMAGE_RGB, OB_F32, nullptr, image.data(), image.dimension(0), image.dimension(1), update_state);
    }
    void update(RgbImageRef<double> image, bool update_state = true) {
        p_.run(OB_IMAGE_RGB, OB_F64, nullptr, image.data(), image.dimension(0), image.dimension(1), update_state);
    }
    /// float16 RGB in (f16_bits_to_f32_bits_fast_nan_zero), float RGB out
    void update(RgbImageRef<const float16_t> input, RgbImageRef<float> out, bool update_state = true) {
        p_.run(OB_IMAGE_RGB_F16, OB_F32, input.data(), out.data(), input.dimension(0), input.dimension(1),
               update_state);
    }
    /// the state (lo_, hi_, lo_state_, hi_state_, counter_, initialized_); not in the reference, for inspection
    ob_image_state state() const { return p_.state(); }

   private:
    impl::ImageProc p_;
};

/// Corrects beam uniformity by minimising the median difference between rows (image_processing.cpp:407-506).
class BeamUniformityCorrector {
   public:
    BeamUniformityCorrector() : p_(OB_IMAGE_BEAM_UNIFORMITY, 0.0, 0.0, 8, 0.92, 0.0, false) {}
    void update(ArrayRef<float> image, bool update_state = true) {
        p_.run(OB_IMAGE_MONO, OB_F32, nullptr, image.data(), image.rows(), image.cols(), update_state);
    }
    void update(ArrayRef<double> image, bool update_state = true) {
        p_.run(OB_IMAGE_MONO, OB_F64, nullptr, image.data(), image.rows(), image.cols(), update_state);
    }
    /// the counter and dark_count_ (up to cap values into dark_count); not in the reference, for inspection
    ob_image_state state(double* dark_count = nullptr, size_t cap = 0) const { return p_.state(dark_count, cap); }

   private:
    impl::ImageProc p_;
};

/// CLAHE-based tone mapping of RGB images (image_processing.cpp:508-710).
class LocalToneMapper {
   public:
    LocalToneMapper() : LocalToneMapper(0.0, 0.2, 1, 0.3, 0.2, true) {}
    LocalToneMapper(int update_every) : LocalToneMapper(0.0, 0.2, update_every, 0.3, 0.2, true) {}
    LocalToneMapper(double lo_percentile, double hi_percentile, int update_every, double damping, bool compress_dr,
                    bool color_correct)
        : LocalToneMapper(lo_percentile, hi_percentile, update_every, damping, compress_dr ? 0.2 : 0.0,
                          color_correct) {}
    LocalToneMapper(double lo_percentile, double hi_percentile, int update_every, double damping,
                    double compress_dr_max_lum, bool color_correct)
        : p_(OB_IMAGE_LOCAL_TONE_MAP, lo_percentile, hi_percentile, update_every, damping, compress_dr_max_lum,
             color_correct) {}

    void update(RgbImageRef<float> image, bool update_state = true) {
        p_.run(OB_IMAGE_RGB, OB_F32, nullptr, image.data(), image.dimension(0), image.dimension(1), update_state);
    }
    void update(RgbImageRef<double> image, bool update_state = true) {
        p_.run(OB_IMAGE_RGB, OB_F64, nullptr, image.data(), image.dimension(0), image.dimension(1), update_state);
    }
    void update(RgbImageRef<const float16_t> input, RgbImageRef<float> output, bool update_state = true) {
        p_.run(OB_IMAGE_RGB_F16, OB_F32, input.data(), output.data(), input.dimension(0), input.dimension(1),
               update_state);
    }
    ob_image_state state() const { return p_.state(); }

   private:
    impl::ImageProc p_;
};

}  // namespace image
}  // namespace core
}  // namespace sdk
}  // namespace ouster
