// c_abi_internal.h — entry points shared between the translation units of libgyroflow_cuda.so, NOT exported
// (the library is built with -fvisibility=hidden; only GF_API symbols leave it).
#pragma once
#include <cstddef>
#include <cstdint>
#include "../../include/gyroflow_cuda.h"

namespace gf {

// Trust verdict of a matrix table (rows of GF_MATRIX_STRIDE floats), as the packed warp kernel wants it: 0 = trusted, TBL_WILD = an
// entry of columns 0-8 is not tame (below), TBL_IBIS = an entry of columns 9-13 (IBIS / OIS shifts) is non-zero.
enum : uint32_t { TBL_WILD = 1u, TBL_IBIS = 2u };
// "tame": zero, or 2^-40 <= |v| <= 2^40 — the magnitudes for which the packed kernel's unguarded numerators are safe
__host__ __device__ __forceinline__ bool tame(float v) { const float a = fabsf(v); return v == 0.0f || (a >= 0x1p-40f && a <= 0x1p40f); }
__host__ __device__ __forceinline__ uint32_t table_entry_verdict(unsigned col, float v) {
    return col < 9u ? (tame(v) ? 0u : TBL_WILD) : (v == 0.0f ? 0u : TBL_IBIS);
}
__host__ __device__ __forceinline__ uint32_t table_row_verdict(const float* r) {
    uint32_t f = 0;
    for (unsigned i = 0; i < GF_MATRIX_STRIDE; ++i) f |= table_entry_verdict(i, r[i]);
    return f;
}

} // namespace gf

// One frame through the warp with a DEVICE matrix table + verdict word, never synchronising: HOST image buffers (page-locked) are
// copied on `cu_stream` before / after the kernel.  `checksum_dev` (nullable): the output buffer's checksum is accumulated into it
// on the same stream, between the kernel and the device-to-host copy.  Used by the render queue.
int gf_internal_run_frame(gf_cuda_ctx* ctx, const gf_buffer_desc* in, const gf_buffer_desc* out, const gf_kernel_params* params,
                          const float* matrices_dev, size_t matrix_rows, const float* mesh_dev, size_t mesh_len,
                          const uint32_t* table_flags_dev, void* cu_stream, uint64_t* checksum_dev);

// Preview overlays (overlay.cu): draw_pixel + draw_safe_area of opencl_undistort.cl:109-154 as a pass over a DEVICE buffer.
// count / scalar: channels and scalar kind (0 u8, 1 u16, 2 f32, 3 f16) of the pixel type.
int gf_internal_draw_overlays(void* cu_stream, uint8_t* buf_dev, size_t len, int width, int height, int stride, const gf_kernel_params* p,
                              int count, int scalar, int is_input, const uint8_t* drawing_dev, size_t drawing_len);
