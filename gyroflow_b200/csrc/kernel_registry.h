// kernel_registry.h — ahead-of-time kernel family: one instantiation per
// (lens model, digital lens, pixel layout, interpolation).  The reference selects its kernel by
// splicing lens-model source text into the OpenCL/WGSL program at run time (gpu/opencl.rs:184-211);
// here every valid combination is compiled for sm_90a up front and looked up by id.
#pragma once
#include "warp_kernel_x2.cuh"

#ifndef GF_X2_MINB
#define GF_X2_MINB 4      // resident 256-thread blocks per SM the packed kernel is compiled for (register cap 65536 / (256 * MINB))
#endif

namespace gf {

typedef void (*KernelFn)(const WarpArgs);

// pixel layouts: (COUNT, SCALAR) pairs that exist in pixel_formats.rs
enum {
    LAY_1U8 = 0, LAY_2U8, LAY_3U8, LAY_4U8,
    LAY_1U16, LAY_2U16, LAY_3U16, LAY_4U16,
    LAY_1F32, LAY_4F32, LAY_4F16,
    LAY_COUNT
};

// the instantiations of one (lens model, digital lens, pixel layout)
// general: every per-frame feature tested at run time; lean: the rare ones compiled out (F_GENERAL_ONLY); packed: two pixels per
// thread (warp_kernel_x2.cuh) where the lens model has a packed form, trusted-table and guarded path picked from the device word
// WarpArgs::table_flags; packed coordinates: the packed kernel writing pass 1 of the two-pass path, one per lens model for every layout
enum KernelVariant { KV_GENERAL, KV_LEAN, KV_PACKED, KV_PACKED_COORDS, KV_COUNT };

// implemented once per lens model in inst_<model>.cu; returns nullptr for combinations that are not compiled
KernelFn gf_kernel_opencv_fisheye(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_opencv_standard(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_poly3(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_poly5(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_ptlens(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_insta360(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_sony(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_generic_polynomial(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_kernel_gopro(int digital, int layout, int interp, KernelVariant v);
KernelFn gf_shade_kernel(int layout);      // pass 2 of the multi-plane mode (shade_kernel.cu)

// The resamplers the library accepts.  Only bilinear is fused into the warp kernels; bicubic, Lanczos4 and EWA CubicBC (Robidoux
// sharp / Robidoux / Mitchell / Catmull-Rom) run the scalar kernels' coordinate pass and then the sampling pass (sample_high_order).
inline bool interp_supported(int interp) {
    return interp == GF_INTERP_BILINEAR || interp == GF_INTERP_BICUBIC || interp == GF_INTERP_LANCZOS4 ||
           (interp >= GF_INTERP_ROBIDOUX_SHARP && interp <= GF_INTERP_CATMULL_ROM);
}

template <int LENS, int DIGITAL, class PIX>
static KernelFn pick_variant(int interp, KernelVariant v) {
    if (!interp_supported(interp)) return nullptr;
    // packed digital lenses: superview, superview6, hyperview (fisheye pairs) and digital_stretch (every packed lens model)
    constexpr bool kPacked = Lens2<LENS>::kHas && Digital2<DIGITAL>::kHas;
    // case order = the order the instantiations reach ptxas, which can shift its instruction scheduling: keep it
    switch (v) {
    case KV_PACKED_COORDS: if constexpr (kPacked) return warp_kernel_x2<LENS, DIGITAL, Pix<1, SC_U8>, GF_X2_MINB, true>; else return nullptr;
    // 4 resident blocks per SM (64 registers, no spills): on H100 3 % faster than 6 (40 registers, ~110 B of spills), the same as 5
    case KV_PACKED: if constexpr (kPacked) if (interp == GF_INTERP_BILINEAR) return warp_kernel_x2<LENS, DIGITAL, PIX, GF_X2_MINB>;
        return nullptr;
    case KV_LEAN:    return warp_kernel<LENS, DIGITAL, PIX, false>;
    case KV_GENERAL: return warp_kernel<LENS, DIGITAL, PIX, true>;
    default: return nullptr;
    }
}
template <int LENS, int DIGITAL>
static KernelFn pick_layout(int layout, int interp, KernelVariant v) {
    switch (layout) {
    case LAY_1U8:  return pick_variant<LENS, DIGITAL, Pix<1, SC_U8>>(interp, v);
    case LAY_2U8:  return pick_variant<LENS, DIGITAL, Pix<2, SC_U8>>(interp, v);
    case LAY_3U8:  return pick_variant<LENS, DIGITAL, Pix<3, SC_U8>>(interp, v);
    case LAY_4U8:  return pick_variant<LENS, DIGITAL, Pix<4, SC_U8>>(interp, v);
    case LAY_1U16: return pick_variant<LENS, DIGITAL, Pix<1, SC_U16>>(interp, v);
    case LAY_2U16: return pick_variant<LENS, DIGITAL, Pix<2, SC_U16>>(interp, v);
    case LAY_3U16: return pick_variant<LENS, DIGITAL, Pix<3, SC_U16>>(interp, v);
    case LAY_4U16: return pick_variant<LENS, DIGITAL, Pix<4, SC_U16>>(interp, v);
    case LAY_1F32: return pick_variant<LENS, DIGITAL, Pix<1, SC_F32>>(interp, v);
    case LAY_4F32: return pick_variant<LENS, DIGITAL, Pix<4, SC_F32>>(interp, v);
    case LAY_4F16: return pick_variant<LENS, DIGITAL, Pix<4, SC_F16>>(interp, v);
    default: return nullptr;
    }
}

} // namespace gf
