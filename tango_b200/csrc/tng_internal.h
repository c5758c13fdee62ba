// tng_internal.h — host-side helpers shared by the translation units of libtango_b200.so.
#pragma once
#include <cuda_runtime.h>
#include <cuda.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/tango_b200.h"

namespace tng {
int set_error(int code, const char* fmt, ...);
int num_sms();
void count_launch();
// Grid of an elementwise kernel over `total` items: one item per thread up to 16 CTAs per SM, then the threads stride
inline int grid_for(long long total, int block = 256) {
  long long g = (total + block - 1) / block;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return static_cast<int>(g);
}
// Encode a bf16 tiled tensor map with SWIZZLE_128B and zero OOB fill (driver entry point resolved at run time so
// the library loads on machines without libcuda).
int encode_tmap_bf16(CUtensorMap* out, const void* ptr, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                     const uint32_t* box);
// The same for rows of a [batch][L][ld] bf16 tensor, read in boxes of 64 columns x `rows` rows of one batch entry.
int encode_tmap_rows_bf16(CUtensorMap* out, const void* ptr, long long ld, long long L, long long batch, uint32_t rows);
// col_stats[(n * C + c) * 2 + {0, 1}] += sum / sum of squares of x[n, :, c] over the HW pixels of image n (x: [NB*HW, ld],
// fp32 or bf16). The per-channel form of the GroupNorm statistics: any grouping (also across a channel concat) is a sum
// of channels. Used when a GEMM cannot emit the statistics from its epilogue (partial tiles, split-K).
int launch_col_stats(const void* x, int dt, long long C, long long ld, long long NB, long long HW, double* col_stats,
                     cudaStream_t st);
// Call right after every kernel launch: counts it (tng_launch_count) and reports a launch error.
inline int check_launch(const char* what) {
  count_launch();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(TNG_ECUDA, "%s launch: %s", what, cudaGetErrorString(e));
  return TNG_OK;
}
// Raise Kernel's dynamic shared-memory limit to `bytes`, once per kernel (the flag is keyed on the kernel itself:
// the gemm_tc_kernel<BN> instantiations share one function type but need different limits).
template <auto Kernel>
int set_max_dynamic_smem(int bytes, const char* what) {
  static bool done = false;
  if (!done) {
    cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e != cudaSuccess) return set_error(TNG_ECUDA, "cudaFuncSetAttribute(%s): %s", what, cudaGetErrorString(e));
    done = true;
  }
  return TNG_OK;
}
}  // namespace tng
