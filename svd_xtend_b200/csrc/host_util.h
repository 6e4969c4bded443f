// Host-side helpers shared by the C-ABI launchers (error reporting, TMA descriptor encode).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

int svdx_fail(int code, const char* msg);
int svdx_fail_cuda(cudaError_t e, const char* what);
// bf16 tiled tensor map, 128-byte swizzle, zero OOB fill. strides[] are bytes for dims 1..rank-1.
int svdx_make_tmap(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                   const uint32_t* box);
// general form: f32 != 0 -> fp32 elements; swizzle_bytes in {0, 32, 64, 128}
int svdx_make_tmap_ex(CUtensorMap* out, const void* base, int f32, int swizzle_bytes, int rank, const uint64_t* dims,
                      const uint64_t* strides, const uint32_t* box);
// bf16 im2col tensor map of a channels-last image tensor, dims {C, W, H, images}, strides[] bytes for dims 1..3:
// 64 channels per pixel, `pixels_per_column` consecutive pixels per load, 128-byte swizzle, zero OOB fill. The start
// pixels span the 3x3 / padding-1 box (corners -1, -1), so a load at start (w - 1, h - 1, n) with offsets (dw + 1, dh + 1)
// reads the pixels of output (n, h, w) onwards shifted by the tap (dw, dh), crossing image rows and images.
int svdx_make_tmap_im2col(CUtensorMap* out, const void* base, const uint64_t* dims, const uint64_t* strides, int pixels_per_column);
extern "C" int svdx_num_sms(void);
// index of the calling thread's current CUDA device (0 when the runtime cannot tell), clamped to [0, 64):
// function attributes such as the dynamic shared-memory limit are per device, so "set once" flags are arrays of this size
int svdx_device_slot(void);
#define SVDX_MAX_DEVICES 64

#define SVDX_CHECK_LAUNCH(what)                                   \
  do {                                                            \
    cudaError_t e__ = cudaGetLastError();                         \
    if (e__ != cudaSuccess) return svdx_fail_cuda(e__, what);     \
  } while (0)
