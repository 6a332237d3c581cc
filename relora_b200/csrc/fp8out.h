// Optional E4M3 side output of a producer kernel (fp8 frozen-weight path): q = sat_e4m3(value * *inv_scale) written next to the
// bf16 result, amax(|value|) recorded for the next micro-step's delayed scale.  Plain struct shared by host and device code.
#pragma once
#include <stdint.h>

namespace rb {

struct Fp8Out {
  uint8_t* q = nullptr;
  long long ld = 0;
  const float* inv_scale = nullptr;
  float* amax = nullptr;
};

// Optional MXFP8 side output of a producer kernel (fused executor on packed weights): the bytes and blocked scales
// mx_quantize_rows would write for the bf16 result, rows < M only.  kg: 128-column groups per row (K rounded up to 128).
struct MxOut {
  uint8_t* q = nullptr;
  long long ld = 0;
  uint8_t* sf = nullptr;
  int kg = 0;
};

}  // namespace rb
