/* Driver of the reference's FailureDetector (recovery_behaviors.cpp, compiled unmodified next to this file by
 * ref_recovery.mk): test infrastructure for tests/test_reference_pin_recovery.py, nothing in the product loads it. */
#include <teb_local_planner/recovery_behaviors.h>

#include <cstdint>

using teb_local_planner::FailureDetector;

extern "C" {

/* FailureDetector with setBufferLength(capacity), fed twists[t] = (linear.x, angular.z) for t = 0 .. T - 1 through
 * update(); osc_out[t] = isOscillating() after step t */
void teb_ref_failure_detector(int32_t capacity, const double* twists, int32_t T, double v_max, double v_backwards_max,
                              double omega_max, double v_eps, double omega_eps, int32_t* osc_out) {
  FailureDetector d;
  d.setBufferLength(capacity);
  for (int32_t t = 0; t < T; ++t) {
    geometry_msgs::Twist tw;
    tw.linear.x = twists[2 * t];
    tw.angular.z = twists[2 * t + 1];
    d.update(tw, v_max, v_backwards_max, omega_max, v_eps, omega_eps);
    osc_out[t] = d.isOscillating() ? 1 : 0;
  }
}

}  /* extern "C" */
