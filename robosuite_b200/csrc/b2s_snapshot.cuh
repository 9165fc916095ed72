// Whole-environment snapshots (b2s_snapshot / b2s_restore): copies between an environment's rows of the handle's per-environment
// arrays and one opaque byte row per environment.  One warp per row; the section table lives in device memory (not the constant bank,
// so the descriptors every other kernel reads are untouched).  Precision-agnostic: sections are counted in 4-byte words.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

// one section of a snapshot row: `words` 4-byte words per environment at ptr + env * stride (bytes), stored from word `off` of the
// row (16-byte aligned); the row words off + words .. off + span are padding, written as zeros so that equal states give equal rows.
// vec: ptr, stride and words allow 16-byte copies.  ptr null (no GJK cache): written as zeros, not restored.
struct SnapSec { char* ptr; long long stride; int off, words, span, vec; };
#define SNAP_IDX 960  // environment indices per launch of snapshot_list_kernel (they travel as a kernel argument)
struct SnapIdx { int idx[SNAP_IDX]; };

__device__ __forceinline__ void snap_gather(const SnapSec* __restrict__ tab, int nsec, uint32_t* __restrict__ row, int e, int lane) {
  for (int k = 0; k < nsec; k++) {
    const SnapSec t = tab[k];
    uint32_t* dst = row + t.off;
    for (int i = (t.ptr ? t.words : 0) + lane; i < t.span; i += 32) dst[i] = 0u;
    if (!t.ptr) continue;
    const char* src = t.ptr + (long long)e * t.stride;
    if (t.vec) {
      const uint4* s4 = (const uint4*)src;
      uint4* d4 = (uint4*)dst;
      for (int i = lane; i < (t.words >> 2); i += 32) d4[i] = s4[i];
    } else {
      const uint32_t* s1 = (const uint32_t*)src;
      for (int i = lane; i < t.words; i += 32) dst[i] = s1[i];
    }
  }
}

// row r <- environment r (all environments in order)
__global__ void __launch_bounds__(256) snapshot_kernel(const SnapSec* __restrict__ tab, int nsec, int row_words, unsigned char* __restrict__ rows,
                                                       int n_rows) {
  const int r = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  snap_gather(tab, nsec, (uint32_t*)rows + (size_t)r * row_words, r, lane);
}

// rows first .. first + n - 1 <- environments ix.idx[0 .. n) (validated on the host)
__global__ void __launch_bounds__(256) snapshot_list_kernel(const SnapSec* __restrict__ tab, int nsec, int row_words, unsigned char* __restrict__ rows,
                                                            int first, int n, SnapIdx ix) {
  const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (w >= n) return;
  snap_gather(tab, nsec, (uint32_t*)rows + (size_t)(first + w) * row_words, ix.idx[w], lane);
}

// environment e <- row src[e] (src null: row e).  -1 leaves the environment untouched; any other index outside [0, n_rows) leaves it
// untouched too and sets warn bit 256.
__global__ void __launch_bounds__(256) restore_kernel(const SnapSec* __restrict__ tab, int nsec, int row_words, const unsigned char* __restrict__ rows,
                                                      int n_rows, const int* __restrict__ src, int n_env, int* __restrict__ warn) {
  const int e = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (e >= n_env) return;
  const int r = src ? src[e] : e;
  if (r == -1) return;
  if (r < -1 || r >= n_rows) {
    if (lane == 0) warn[e] |= 256;
    return;
  }
  const uint32_t* row = (const uint32_t*)rows + (size_t)r * row_words;
  for (int k = 0; k < nsec; k++) {
    const SnapSec t = tab[k];
    if (!t.ptr) continue;
    const uint32_t* s1 = row + t.off;
    char* dst = t.ptr + (long long)e * t.stride;
    if (t.vec) {
      const uint4* s4 = (const uint4*)s1;
      uint4* d4 = (uint4*)dst;
      for (int i = lane; i < (t.words >> 2); i += 32) d4[i] = s4[i];
    } else {
      uint32_t* d1 = (uint32_t*)dst;
      for (int i = lane; i < t.words; i += 32) d1[i] = s1[i];
    }
  }
}
