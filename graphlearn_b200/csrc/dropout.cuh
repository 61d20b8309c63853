// Dropout mask of the fused GraphSAGE trainer's hidden layers, shared by the forward epilogue (sage_fused.cu) and the
// batch-norm apply kernel (sage_bn.cu), so that both draw bit-identical masks.
#pragma once
#include "common.cuh"

namespace glb {

// Dropout mask bits of row `row` of a layer's output: ONE Philox4x32-10 call (key = seed, counter = (row,
// layer << 24 | col / 32 * 4 + col / 2 % 4, step counter low, high word)) gives the 16 bits of the eight columns
// {32 (col / 32) + 8 w + 2 (col / 2 % 4) + e : w < 4, e < 2}: word w, low half for e = 0, high half for e = 1.  These
// are exactly the eight columns one lane of the forward epilogue holds in a row of a 32-column slice, so a lane draws
// once per row and slice and the mask does not depend on the tile schedule, the CTA or the image that computes the
// column.  `state` = {seed, step counter}, 16-byte aligned.  An element is kept when its 16 bits are >= round(p * 65536).
__device__ __forceinline__ uint4 dropout_philox(const unsigned long long* state, uint32_t layer, uint32_t row, uint32_t col) {
  const ulonglong2 st = *reinterpret_cast<const ulonglong2*>(state);
  return Philox(st.x)(row, (layer << 24) | ((col >> 5) << 2) | ((col >> 1) & 3u), (uint32_t)st.y, (uint32_t)(st.y >> 32));
}

}  // namespace glb
