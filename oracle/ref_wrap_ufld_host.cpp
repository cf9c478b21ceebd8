// ref_wrap_ufld_host.cpp -- TEST INFRASTRUCTURE.  CPU-only wrapper around UFLD's driver compiled where it lies (oracle/Makefile:
// -Dmain=ref_ufld_driver_main, against oracle/shim_ufld): its own argmax and softmax_mul, called with the test's arguments.
#include <type_traits>

#include "lane_det.cpp"

#define REF_API __attribute__((visibility("default")))

extern "C" {
REF_API void ref_ufld_argmax(float* x, float* y, int rows, int cols, int chan) { argmax(x, y, rows, cols, chan); }
REF_API void ref_ufld_softmax_mul(float* x, float* y, int rows, int cols, int chan) { softmax_mul(x, y, rows, cols, chan); }
// 1 when the driver's unqualified exp(float) resolves to the float overload (std::exp, expf) with this build's includes, 0
// when it is the C library's double exp
REF_API int ref_ufld_exp_is_float(void) { return std::is_same<decltype(exp(1.0f)), float>::value ? 1 : 0; }
}
