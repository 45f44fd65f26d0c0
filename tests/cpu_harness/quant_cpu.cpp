// CPU harness (TEST INFRASTRUCTURE) around the RGBA8 quantiser of animate3d_b200/csrc/a3d_raster_math.h, the arithmetic
// the forward-only RGBA8 render kernel applies to every pixel.
// Build: g++ -O1 -ffp-contract=off -shared -fPIC quant_cpu.cpp -o quant_cpu.so   (done by tests/test_visualize_cpu.py)
#include "../../animate3d_b200/csrc/a3d_raster_math.h"

extern "C" {

// out[i] = quantise_u8(in[i]); with clamp != 0, quantise_u8(clamp01(in[i])) (the colour channels)
void quant_cpu(const float* in, uint8_t* out, long n, int clamp) {
  for (long i = 0; i < n; ++i) out[i] = a3d::quantise_u8(clamp ? a3d::clamp01(in[i]) : in[i]);
}

}
