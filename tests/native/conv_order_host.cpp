// Host build of the conv2 weight-gradient reduction order (tfy_conv_index.cuh: c_wg_slice), for
// tests/test_conv2_wgrad_order.py.
#include "tfy_conv_index.cuh"

extern "C" void tfy_host_wg_slice(int total4, int n_part, int owner, int threads, int* out) {
    const CWgSlice s = c_wg_slice(total4, n_part, owner, threads);
    out[0] = s.lo;
    out[1] = s.len;
    out[2] = s.parts;
    out[3] = c_wg_per(total4, n_part);
}
