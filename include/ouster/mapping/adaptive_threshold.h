// adaptive_threshold.h -- AdaptiveThreshold (mirrors ouster_mapping/include/ouster/mapping/adaptive_threshold.h and
// ouster_mapping/src/adaptive_threshold.cpp).  Host scalars that turn each ICP correction into the next
// align_points_to_map call's max_distance; nothing here runs on the GPU.  The rotation angle is Eigen::AngleAxisd's:
// the rotation matrix converted to a quaternion (Eigen's trace / largest-diagonal rule), then 2 atan2(|vec|, |w|).
#pragma once
#include <cmath>
#include <limits>

#include "ouster/core/typedefs.h"

namespace ouster {
namespace sdk {
namespace mapping {

struct AdaptiveThreshold {
    explicit AdaptiveThreshold(double max_range, double initial_threshold = 2.0, double min_motion_threshold = 0.01)
        : min_motion_threshold_(min_motion_threshold),
          max_range_(max_range),
          model_sse_(initial_threshold * initial_threshold),
          num_samples_(1) {}

    /// adaptive_threshold.cpp: model_error = |t| + 2 max_range sin(theta / 2), counted when above the minimum motion
    void update_model_deviation(const core::Matrix4dR& current_deviation) {
        const double theta = rotation_angle(current_deviation);
        const double delta_rot = 2.0 * max_range_ * std::sin(theta / 2.0);
        const double tx = current_deviation(0, 3), ty = current_deviation(1, 3), tz = current_deviation(2, 3);
        const double delta_trans = std::sqrt((tx * tx + ty * ty) + tz * tz);
        const double model_error = delta_trans + delta_rot;
        if (model_error > min_motion_threshold_) {
            model_sse_ += model_error * model_error;
            num_samples_++;
        }
    }

    /// the KISS-ICP adaptive threshold used in registration
    double compute_threshold() const { return std::sqrt(model_sse_ / num_samples_); }

    static double rotation_angle(const core::Matrix4dR& r) {
        double w, v[3];
        const double t = r(0, 0) + r(1, 1) + r(2, 2);
        if (t > 0) {
            double s = std::sqrt(t + 1.0);
            w = 0.5 * s;
            s = 0.5 / s;
            v[0] = (r(2, 1) - r(1, 2)) * s;
            v[1] = (r(0, 2) - r(2, 0)) * s;
            v[2] = (r(1, 0) - r(0, 1)) * s;
        } else {
            int i = 0;
            if (r(1, 1) > r(0, 0)) i = 1;
            if (r(2, 2) > r(i, i)) i = 2;
            const int j = (i + 1) % 3, k = (i + 2) % 3;
            double s = std::sqrt(r(i, i) - r(j, j) - r(k, k) + 1.0);
            v[i] = 0.5 * s;
            s = 0.5 / s;
            w = (r(k, j) - r(j, k)) * s;
            v[j] = (r(j, i) + r(i, j)) * s;
            v[k] = (r(k, i) + r(i, k)) * s;
        }
        const double n = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
        return n < std::numeric_limits<double>::epsilon() ? 0.0 : 2.0 * std::atan2(n, std::fabs(w));
    }

    double min_motion_threshold_;
    double max_range_;
    double model_sse_;
    int num_samples_;
};

}  // namespace mapping
}  // namespace sdk
}  // namespace ouster
