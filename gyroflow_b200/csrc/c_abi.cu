// c_abi.cu — extern "C" boundary of the CUDA backend (include/gyroflow_cuda.h).
//
// Mirrors the reference's backend-wrapper life cycle:
//   gf_cuda_create          <- OclWrapper::new        src/core/gpu/opencl.rs:178  (WgpuWrapper::new wgpu.rs:147)
//   gf_cuda_undistort_image <- OclWrapper::undistort_image opencl.rs:330-448 (wgpu.rs:454-559)
//   gf_cuda_destroy         <- Drop / clear_gpu_cache_current_thread  stabilization/mod.rs:72-81
// plus the validation `Stabilization::process_pixels` performs before dispatch (stabilization/mod.rs:612-640).
// There is no CPU fallback: without a usable CUDA device every compute call fails with GF_ERR_CUDA.
#include <cuda_runtime.h>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <mutex>
#include <cmath>
#include <algorithm>
#include <string>
#include <vector>

#include "kernel_registry.h"
#include "c_abi_internal.h"
#include "gyro_dev.h"
#include <nvtx3/nvToolsExt.h>

using namespace gf;

namespace {

struct Slot {                                   // one in-flight set of per-frame tables
    GrowBuf<float, true> h_mat, h_mesh;
    GrowBuf<float> d_mat, d_mesh;
    GrowBuf<double> d_mesh64;                   // the mesh widened to f64 once per frame (cpu_undistort.rs:539), then one MeshAux
    Event done;
};
constexpr int kSlots = 4;
constexpr int kPackedBlockY = 4;                // packed-kernel blocks are GF_BLOCK_X x kPackedBlockY threads
constexpr unsigned long long kMaxOutRows = 65535ull * GF_BLOCK_Y;   // output rows one launch covers (65535 row blocks, gridDim.y)
static_assert(2 * kPackedBlockY == GF_BLOCK_Y, "the packed kernel's row blocks cover GF_BLOCK_Y rows, like the scalar kernels'");

// Per pixel layout (LAY_*): bytes per pixel, channels, scalar kind (SC_*), the maximum value pixel_value_limit is compared against
struct LayoutInfo { int bpp, channels, scalar; float max_value; };
constexpr LayoutInfo kLayouts[LAY_COUNT] = {
    { 1, 1, SC_U8,  255.0f },          { 2, 2, SC_U8,  255.0f },          { 3, 3, SC_U8,  255.0f },   { 4, 4, SC_U8,  255.0f },
    { 2, 1, SC_U16, 65535.0f },        { 4, 2, SC_U16, 65535.0f },        { 6, 3, SC_U16, 65535.0f }, { 8, 4, SC_U16, 65535.0f },
    { 4, 1, SC_F32, 3.402823466e38f }, { 16, 4, SC_F32, 3.402823466e38f }, { 8, 4, SC_F16, 3.402823466e38f },
};

// What the uniforms and the kernel choice of a frame depend on besides the frame: lens, digital lens, layout, and the compiled kernels
// by variant.  GF_DISABLE_X2 (no packed kernel) and GF_DISABLE_FILTER (no filtered pre-pass) take a fast path out of service for A/B
// comparisons; GF_DISABLE_LEAN (no lean and no packed kernel) makes every frame run the general kernel, so that its instantiations can
// be checked on plain frames.  They are read whenever a combo is made: once per context, and on every gf_cuda_plan /
// gf_combo_supported query.
struct Combo {
    int lens = 0, digital = 0, layout = 0;
    KernelFn kernels[KV_COUNT] = {};     // nullptr where not compiled (or switched off)
    bool no_filter = false;
    int bpp() const { return kLayouts[layout].bpp; }
};

} // namespace

struct gf_cuda_ctx {
    int device = 0;
    Combo combo;
    int interpolation = 0;
    int width = 0, height = 0, output_width = 0, output_height = 0;    // Stabilization.size / output_size
    KernelFn fn_shade = nullptr;         // pass 2 of the two-pass path
    GrowBuf<uint32_t> const_flags;       // two device words {0, 1}: the verdict of the host scan of host tables, as the kernel wants it
    GrowBuf<uint32_t> vflags;            // scratch verdict word of gf_cuda_validate_tables_dev
    // Every call is ordered after the previous one on the device, whatever streams they name: `last_call` is recorded at the end of each
    // call, and a call on another stream than `last_stream` waits for it first (order_after_last_call).  The calls share the state
    // below (deferred-pair queue and counters, coordinate maps, staging), and gf_cuda_synchronize waits for `last_stream` only.
    cudaStream_t last_stream = nullptr;
    Event last_call;
    FilterPrepass filter;
    // preview overlays (overlay.cu), off unless gf_cuda_set_overlays: device copy of the drawing buffer, private copy of a DEVICE input
    int overlays = 0;
    GrowBuf<uint8_t, true> h_drawing;
    GrowBuf<uint8_t> d_drawing, src_ovl;
    PlaneStaging plane_staging;          // device copies of HOST planes, one plane's worth from gf_cuda_create on
    // The longest HOST input / output (0: none) a single-plane call takes: the lengths of gf_cuda_create's buffers, like the reference's
    // fixed OpenCL buffers.  gf_cuda_undistort_planes grows the staging instead, which leaves these limits alone.
    size_t host_in_len = 0, host_out_len = 0;
    GrowBuf<uint2> coords;               // two-pass path: the frame's coordinate map(s)
    Stream stream;
    size_t max_rows = 0;
    Slot slots[kSlots];
    int next_slot = 0;
    unsigned long long launches = 0;
    std::string last_error;
};

namespace {

// LAY_* of a pixel type (GF_PIX_*), or -1 if unknown
int pix_layout(int pixel_type) {
    static constexpr int kPixLayout[GF_PIX_COUNT] = { LAY_1U8, LAY_1U16, LAY_3U8, LAY_4U8, LAY_4U8, LAY_3U16, LAY_4U16, LAY_4U16,
                                                      LAY_4F32, LAY_4F16, LAY_1F32, LAY_2U8, LAY_2U16 };
    return (pixel_type >= 0 && pixel_type < GF_PIX_COUNT) ? kPixLayout[pixel_type] : -1;
}

KernelFn find_kernel(const Combo& c, int interp, KernelVariant v) {
    switch (c.lens) {
    case GF_LENS_OPENCV_FISHEYE:     return gf_kernel_opencv_fisheye(c.digital, c.layout, interp, v);
    case GF_LENS_OPENCV_STANDARD:    return gf_kernel_opencv_standard(c.digital, c.layout, interp, v);
    case GF_LENS_POLY3:              return gf_kernel_poly3(c.digital, c.layout, interp, v);
    case GF_LENS_POLY5:              return gf_kernel_poly5(c.digital, c.layout, interp, v);
    case GF_LENS_PTLENS:             return gf_kernel_ptlens(c.digital, c.layout, interp, v);
    case GF_LENS_INSTA360:           return gf_kernel_insta360(c.digital, c.layout, interp, v);
    case GF_LENS_SONY:               return gf_kernel_sony(c.digital, c.layout, interp, v);
    case GF_LENS_GENERIC_POLYNOMIAL: return gf_kernel_generic_polynomial(c.digital, c.layout, interp, v);
    case GF_LENS_GOPRO:              return gf_kernel_gopro(c.digital, c.layout, interp, v);
    default: return nullptr;
    }
}

bool make_combo(int pixel_type, int lens, int digital, int interp, Combo* c) {
    c->layout = pix_layout(pixel_type); c->lens = lens; c->digital = digital;
    const bool no_lean = getenv("GF_DISABLE_LEAN") != nullptr;
    const bool no_packed = no_lean || getenv("GF_DISABLE_X2") != nullptr;
    c->no_filter = getenv("GF_DISABLE_FILTER") != nullptr;
    for (int v = 0; v < KV_COUNT; ++v)
        c->kernels[v] = ((no_packed && v >= KV_PACKED) || (no_lean && v == KV_LEAN)) ? nullptr : find_kernel(*c, interp, (KernelVariant)v);
    return c->layout >= 0;                                 // false: unknown pixel type
}

const char* const kLensNames[GF_LENS_COUNT] = {
    "none", "opencv_fisheye", "opencv_standard", "poly3", "poly5", "ptlens", "insta360", "sony", "generic_polynomial",
    "gopro", "gopro_superview", "gopro_hyperview", "gopro_warp", "digital_stretch", "gopro6_superview" };

// process_pixels / OclWrapper::new validation (stabilization/mod.rs:613,636-640; opencl.rs:179; wgpu.rs:150)
// `err`: the context's message, or nullptr before there is a context.
int validate(std::string* err, const gf_kernel_params* p, const gf_buffer_desc* in, const gf_buffer_desc* out, int bpp) {
    if (!p || !in || !out) return fail(err, GF_ERR_BAD_PARAMS, "null argument");
    if (in->height < 4 || out->height < 4 || p->height < 4 || p->output_height < 4)
        return fail(err, GF_ERR_SIZE_TOO_SMALL, "SizeTooSmall: height < 4");
    if (p->stride < 1 || p->output_stride < 1) return fail(err, GF_ERR_BAD_STRIDE, "InvalidStride: stride < 1");
    if (p->width > 16384 || p->output_width > 16384 || p->width < 1 || p->output_width < 1)
        return fail(err, GF_ERR_BAD_PARAMS, "width out of range (1..16384)");
    if (in->width > p->stride)         return fail(err, GF_ERR_BAD_STRIDE, "InvalidStride: input width > stride");
    if (out->width > p->output_stride) return fail(err, GF_ERR_BAD_STRIDE, "InvalidStride: output width > output_stride");
    if (p->stride != in->stride || p->output_stride != out->stride)
        return fail(err, GF_ERR_BAD_STRIDE, "InvalidStride: KernelParams stride differs from the buffer description");
    if (p->bytes_per_pixel != bpp) return fail(err, GF_ERR_BAD_PARAMS, "bytes_per_pixel does not match the pixel type");
    if (p->matrix_count < 1) return fail(err, GF_ERR_BAD_PARAMS, "matrix_count < 1");
    if ((in->kind != GF_BUF_HOST && in->kind != GF_BUF_DEVICE) || (out->kind != GF_BUF_HOST && out->kind != GF_BUF_DEVICE) || !in->ptr || !out->ptr)
        return fail(err, GF_ERR_BAD_PARAMS, "unsupported buffer source");
    // every tap the kernel may read must be inside the input buffer (Rust would panic on the slice index)
    const long long x0 = p->source_rect[0], y0 = p->source_rect[1], x1 = x0 + p->source_rect[2], y1 = y0 + p->source_rect[3];
    if (p->source_rect[2] > 0 && p->source_rect[3] > 0) {
        if (x0 < 0 || y0 < 0) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "source_rect has a negative origin");
        const unsigned long long last = (unsigned long long)(y1 - 1) * (unsigned long long)p->stride + (unsigned long long)x1 * (unsigned long long)bpp;
        if (last > in->len) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch input: source_rect exceeds the input buffer");
    }
    if (out->len == 0) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "empty output buffer");
    // launch geometry: at least one whole pixel per row, and ceil(len / output_stride) rows in blocks of GF_BLOCK_Y rows, at most 65535
    // blocks (gridDim.y); checked here so that gf_cuda_plan refuses what the rendering call would
    const unsigned long long out_rows = (out->len + (unsigned long long)p->output_stride - 1) / (unsigned long long)p->output_stride;
    if (p->output_stride < bpp || out_rows > kMaxOutRows)
        return fail(err, GF_ERR_BAD_PARAMS, "output buffer geometry out of range (a pixel per row, at most 524280 rows)");
    return GF_OK;
}

// f32 mesh -> f64 once per frame (cpu_undistort.rs:539) + the per-frame constants of MeshAux, all on the device so that
// device-resident meshes never touch the host.  o has room for GF_MESH_MAX_LEN doubles followed by one MeshAux.
__global__ void widen_mesh_kernel(const float* __restrict__ m, double* __restrict__ o, int n, float width_f, float height_f) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = (double)m[i];
    if (i == 0 && n >= 9) make_mesh_aux(m, width_f, height_f, *reinterpret_cast<MeshAux*>(o + GF_MESH_MAX_LEN));
}
// one block: every thread ORs its rows, the block reduces, thread 0 WRITES the verdict (no prior memset, no atomics on the word)
__global__ void __launch_bounds__(1024) scan_tables_kernel(const float* __restrict__ m, size_t rows, uint32_t* flags) {
    __shared__ unsigned warp_or[32];
    unsigned f = 0;
    const size_t n = rows * GF_MATRIX_STRIDE;
    for (size_t i = threadIdx.x; i < n; i += blockDim.x) f |= table_entry_verdict((unsigned)(i % GF_MATRIX_STRIDE), m[i]);
    f = __reduce_or_sync(0xffffffffu, f);
    if ((threadIdx.x & 31u) == 0u) warp_or[threadIdx.x >> 5] = f;
    __syncthreads();
    if (threadIdx.x < 32u) {
        f = threadIdx.x < (blockDim.x >> 5) ? warp_or[threadIdx.x] : 0u;
        f = __reduce_or_sync(0xffffffffu, f);
        if (threadIdx.x == 0u) *flags = f;
    }
}

// Everything the reference recomputes per pixel from per-frame constants (cpu_undistort.rs:421-528), computed once, on the
// host, with the same IEEE float operations (this TU is built with -ffp-contract=off; sin/cos come from gf_math.cuh, the
// same code the device runs).
// Reads A.p, A.src / A.dst and their lengths, and A.mesh_len.
void fill_uniforms(WarpArgs& A, const Combo& c) {
    const gf_kernel_params* p = &A.p;
    const uint8_t* const src = A.src;
    const uint8_t* const dst = A.dst;
    const int bpp = c.bpp();
    A.out_rows = (int)((A.dst_len + (size_t)p->output_stride - 1) / (size_t)p->output_stride);
    A.out_cols = p->output_stride / bpp;
    const int align = (bpp == 1 || bpp == 2 || bpp == 4 || bpp == 8 || bpp == 16) ? bpp : (bpp == 3 ? 1 : 2);
    uint32_t f = 0;
    if (p->matrix_count > 1) f |= F_RS;
    if ((p->flags & 16) == 16) f |= F_HRS;
    A.r_limit_sq = p->r_limit * p->r_limit;                                      // :521
    if (A.r_limit_sq > 0.0f) f |= F_RLIMIT;
    if (p->light_refraction_coefficient != 1.0f && p->light_refraction_coefficient > 0.0f) f |= F_REFRACT;
    if (A.mesh_len > 0) f |= F_MESH;
    if ((p->flags & 2) == 2 && c.digital != GF_LENS_NONE) f |= F_DIGITAL;
    if (p->input_horizontal_stretch > 0.001f && p->input_horizontal_stretch != 1.0f) f |= F_HSTRETCH;
    if (p->input_vertical_stretch   > 0.001f && p->input_vertical_stretch   != 1.0f) f |= F_VSTRETCH;
    if (p->lens_correction_amount < 1.0f) f |= F_LCA;
    if (p->input_rotation != 0.0f) f |= F_INROT;
    if (p->background_mode == 1) f |= F_BG1;
    if (p->background_mode == 2) f |= F_BG2;
    if (p->background_mode == 3) f |= F_BG3;
    if ((p->flags & 1) == 1) f |= F_FIXRANGE;
    if ((p->flags & 4) == 4) f |= F_FILLBG;
    if (lens_noop(c.lens, p->k)) f |= F_LENS_NOOP;
    if ((reinterpret_cast<uintptr_t>(src) % (uintptr_t)align) == 0 && (p->stride % align) == 0) f |= F_SRC_VEC;
    if ((f & F_SRC_VEC) && (reinterpret_cast<uintptr_t>(src) % 8u) == 0 && (p->stride % 8) == 0 && (A.src_len % 8ull) == 0) f |= F_SRC_VEC8;
    if ((reinterpret_cast<uintptr_t>(dst) % (uintptr_t)align) == 0 && (p->output_stride % align) == 0) f |= F_DST_VEC;
    if ((p->flags & 128) == 128) f |= F_FB_INV;
    if (p->plane_index == 0) f |= F_IS_Y;
    if (p->translation3d[0] != 0.0f || p->translation3d[1] != 0.0f || p->translation3d[2] != 0.0f) f |= F_T3D;
    if (!(p->pixel_value_limit >= kLayouts[c.layout].max_value)) f |= F_PIXLIMIT;
    {   // magnitudes the packed kernel's fast paths rely on (otherwise the scalar lean kernel, which has no such assumptions, runs)
        bool wild = false;
        for (int i = 0; i < 12; ++i) if (!(std::isfinite(p->k[i]) && fabsf(p->k[i]) <= 0x1p40f)) wild = true;
        if (!(fabsf(p->translation2d[0]) < 0x1p19f && fabsf(p->translation2d[1]) < 0x1p19f)) wild = true;
        if (!(tame(p->f[0]) && tame(p->f[1]) && std::isfinite(p->c[0]) && std::isfinite(p->c[1]))) wild = true;
        // packed gopro lens: k1 is a divisor (paraxial guess of the Newton inversion) and the 89-degree cut-off is a literal
        if (c.lens == GF_LENS_GOPRO && (!(tame(p->k[1]) && p->k[1] != 0.0f) || gf_tanf(1.5533f) != 0x1.c9315ap+5f)) wild = true;
        if (c.digital == GF_LENS_GOPRO_WARP) for (int i = 0; i < 16; ++i) if (!(std::isfinite(p->digital_lens_params[i]) && fabsf(p->digital_lens_params[i]) <= 0x1p40f)) wild = true;
        if (wild) f |= F_WILD;
    }
    A.feat = f;

    for (int i = 0; i < 4; ++i) A.bg[i] = p->background[i] * p->max_pixel_value;  // :523
    const float factor = fmaxf(1.0f - p->lens_correction_amount, 0.001f);         // :526
    A.out_c[0] = (float)p->output_width / 2.0f; A.out_c[1] = (float)p->output_height / 2.0f;   // :527
    A.out_f[0] = p->f[0] / p->fov / factor;      A.out_f[1] = p->f[1] / p->fov / factor;        // :528

    A.width_f = (float)p->width; A.height_f = (float)p->height;
    A.frame_w = A.width_f; A.frame_h = A.height_f;
    A.rot_cos = 1.0f; A.rot_sin = 0.0f;
    if (p->input_rotation != 0.0f) {                                              // :485-489 (rotate_point :262-265)
        const float rotation = p->input_rotation * (3.14159274101257324f / 180.0f);
        A.rot_cos = gf_cosf(rotation); A.rot_sin = gf_sinf(rotation);
        const float fx = A.rot_cos * (A.width_f - 0.0f) - A.rot_sin * (A.height_f - 0.0f) + 0.0f;
        const float fy = A.rot_sin * (A.width_f - 0.0f) + A.rot_cos * (A.height_f - 0.0f) + 0.0f;
        A.frame_w = rs_round(fabsf(fx)); A.frame_h = rs_round(fabsf(fy));
    }
    A.omap_x = make_map((float)p->output_rect[0], (float)(p->output_rect[0] + p->output_rect[2]), 0.0f, (float)p->output_width,  (float)A.out_cols);
    A.omap_y = make_map((float)p->output_rect[1], (float)(p->output_rect[1] + p->output_rect[3]), 0.0f, (float)p->output_height, (float)A.out_rows);
    A.smap_x = make_map(0.0f, A.frame_w, (float)p->source_rect[0], (float)(p->source_rect[0] + p->source_rect[2]), -1.0f);
    A.smap_y = make_map(0.0f, A.frame_h, (float)p->source_rect[1], (float)(p->source_rect[1] + p->source_rect[3]), -1.0f);
    A.rs_lim = (p->flags & 16) == 16 ? p->width : p->height;
    A.row_lim = std::min(A.rs_lim, p->matrix_count - 1);
    const float lim = p->pixel_value_limit;
    A.u8_limit = (lim != lim) ? 255 : (lim < 0.0f ? 0 : (lim >= 255.0f ? 255 : (int)lim));
    A.src_rect[0] = p->source_rect[0]; A.src_rect[1] = p->source_rect[1];
    A.src_rect[2] = p->source_rect[0] + p->source_rect[2]; A.src_rect[3] = p->source_rect[1] + p->source_rect[3];
    A.interior_span[0] = A.src_rect[2] - 2 - A.src_rect[0]; A.interior_span[1] = A.src_rect[3] - 2 - A.src_rect[1];
    if (A.interior_span[0] < 0 || A.interior_span[1] < 0 || A.interior_span[0] >= (1 << 17) || A.interior_span[1] >= (1 << 17) || A.rs_lim >= (1 << 22)) { A.interior_span[0] = 0; A.interior_span[1] = 0; A.feat |= F_WILD; }   // no interior at all
    // source-rect maps of the packed kernel (see map_apply_x2): in_min == 0, moderate non-zero scale, divisor <= 2^20, |c| >= 2^-10,
    // source rect inside [0, 2^16) so that every coordinate the rounding shortcut cannot represent is outside the image anyway
    // (in_min must be +0, not -0: map_apply_x2 skips x - in_min)
    auto smap_ok = [](const MapC& m) { return m.fast_div && m.in_min == 0.0f && !std::signbit(m.in_min) && m.mul != 0.0f && tame(m.mul) && m.div > 0.0f && m.div <= 0x1p20f && std::isfinite(m.add) && fabsf(m.add) <= 0x1p16f; };
    if (!(smap_ok(A.smap_x) && smap_ok(A.smap_y) && fabsf(p->c[0]) >= 0x1p-10f && fabsf(p->c[1]) >= 0x1p-10f &&
          A.src_rect[0] >= 0 && A.src_rect[1] >= 0 && A.src_rect[2] <= (1 << 16) && A.src_rect[3] <= (1 << 16))) A.feat |= F_WILD;
    // pixel-index maps of the packed kernel: identity, or a positive moderate scale (map_apply_int_lean in warp_kernel_x2.cuh)
    auto int_map_ok = [](const MapC& m) {
        return m.identity || (m.fast_div && m.mul > 0.0f && m.div > 0.0f && tame(m.mul) && std::isfinite(m.add) && fabsf(m.in_min) <= 0x1p20f);
    };
    if (!(int_map_ok(A.omap_x) && int_map_ok(A.omap_y))) A.feat |= F_WILD;
    // integer prologue of the packed kernel: identity maps -> opx = (x - in_min) + add with integer in_min / add
    // the packed kernel's 8-bit sampler (it only runs without F_WILD: then 0 <= rx0, ry0 <= 2^16 and span < 2^17, far from overflow):
    // the source rect's origin folded into the rounding word and into the gather's base address
    const bool tame_rect = (A.feat & F_WILD) == 0;
    A.hot.wbias[0] = 0x4affffff + (tame_rect ? 64 * A.src_rect[0] : 0); A.hot.wbias[1] = 0x4affffff + (tame_rect ? 64 * A.src_rect[1] : 0);
    A.hot.wlim[0] = 64u * (unsigned)A.interior_span[0] + 63u; A.hot.wlim[1] = 64u * (unsigned)A.interior_span[1] + 63u;
    A.hot.src = tame_rect ? src + ((long long)A.src_rect[1] * (long long)p->stride + (long long)A.src_rect[0] * (long long)bpp) : src;
    A.hot.full = 0;
    if (A.omap_x.identity && A.omap_y.identity && A.omap_x.add == truncf(A.omap_x.add) && A.omap_y.add == truncf(A.omap_y.add) &&
        fabsf(A.omap_x.add) < 0x1p20f && fabsf(A.omap_y.add) < 0x1p20f && fabsf(A.omap_x.in_min) < 0x1p20f && fabsf(A.omap_y.in_min) < 0x1p20f) {
        A.hot.x_off = (int)A.omap_x.add - (int)A.omap_x.in_min; A.hot.y_off = (int)A.omap_y.add - (int)A.omap_y.in_min;
        // :551 — opx >= 0 && (opx as i32) < output_width  <=>  0 <= x + x_off < output_width
        A.hot.x0 = std::max(0, -A.hot.x_off); A.hot.x1 = std::min(A.out_cols, p->output_width - A.hot.x_off);
        A.hot.y0 = std::max(0, -A.hot.y_off); A.hot.y1 = std::min(A.out_rows, p->output_height - A.hot.y_off);
        A.hot.full_rows = (int)std::min<size_t>(A.dst_len / (size_t)p->output_stride, (size_t)A.out_rows);
        const size_t tail = A.dst_len - (size_t)A.hot.full_rows * (size_t)p->output_stride;
        A.hot.last_cols = (A.hot.full_rows < A.out_rows) ? (int)std::min<size_t>(tail / (size_t)bpp, (size_t)A.out_cols) : 0;
        // a last row that holds all of [x0, x1) or none of it is a plain row bound: fold it into y1 and keep the per-pixel test to
        // four compares; only a row cut inside [x0, x1) needs the full_rows / last_cols test (F_SHORTROW)
        if (A.hot.full_rows < A.out_rows) {
            if (A.hot.last_cols >= A.hot.x1) A.hot.y1 = std::min(A.hot.y1, A.hot.full_rows + 1);
            else if (A.hot.last_cols <= A.hot.x0) A.hot.y1 = std::min(A.hot.y1, A.hot.full_rows);
            else A.feat |= F_SHORTROW;
        }
        A.feat |= F_INTPRO;
        // the packed launch (32 x 4 threads of two rows each) covers exactly [0, out_cols) x [0, out_rows), and every pixel of it is written
        auto plus_zero = [](float v) { return v == 0.0f && !std::signbit(v); };
        A.hot.full = (A.feat & (F_WILD | F_SHORTROW)) == 0 && A.hot.x0 == 0 && A.hot.x1 == A.out_cols && A.hot.y0 == 0 && A.hot.y1 == A.out_rows &&
                     A.out_cols % GF_BLOCK_X == 0 && A.out_rows % (2 * kPackedBlockY) == 0 && plus_zero(A.smap_x.add) && plus_zero(A.smap_y.add);
    }
}

// One call through the warp: `FrameJob job{n, in, out, p, matrices, rows, mesh, mesh_len, stream}`, then the options a call needs.
struct FrameJob {
    size_t n; const gf_buffer_desc* in; const gf_buffer_desc* out; const gf_kernel_params* p;   // arrays of the frame's n planes
    const float* matrices; size_t matrix_rows;
    const float* mesh; size_t mesh_len;
    void* stream;                                  // nullptr: the context's stream
    bool tables_on_device = false;                 // matrices / mesh are device pointers (else host memory, staged through a slot)
    bool sync_host = true;                         // with a HOST image buffer: wait for the frame before returning
    int kind = -1; const char* kind_error = nullptr;   // the kind every buffer must have (-1: either), and the refusal's message
    bool grow_staging = false;                     // HOST planes of any length (the staging grows), not only up to gf_cuda_create's
    bool coord_only = false;                       // ST maps: the coordinate pass only, into ctx->coords
    const uint32_t* table_flags_dev = nullptr;     // device tables' verdict word (nullptr: not validated, guarded path)
    const uint8_t* drawing = nullptr; size_t drawing_len = 0;   // preview overlays (after gf_cuda_set_overlays)
};

// How a frame is rendered: the one planner behind run_frame and gf_cuda_plan.
struct Plan {
    bool two_pass;                  // coordinates into a map (pass 1), then one sampling launch per plane (pass 2)
    int n_maps;                     // coordinate maps of pass 1: 1, or 3 for EWA (pixel + two Jacobian probes)
    KernelVariant kernel;           // what renders pass 1 (or the whole frame)
    bool filter;                    // the packed kernel runs the filtered rolling-shutter pre-pass if the lens has a radial table
};
// A holds the frame's filled uniforms; table_flags is what the HOST knows of the matrix table (0 = tame and IBIS-free, non-zero =
// anything else, including device tables not scanned on the host).  n_planes: the planes that share this coordinate pass.
Plan plan_frame(const Combo& c, const WarpArgs& A, uint32_t table_flags, bool tables_on_device, size_t n_planes, bool coord_only) {
    Plan pl;
    // Two-pass mode: used for multi-plane frames, for every resampler other than bilinear (so that the 16/64-tap and EWA code lives in
    // 11 sampling kernels instead of every lens instantiation) and for ST maps (pass 1 only).  EWA needs three coordinate maps.
    const int interp = A.p.interpolation;
    pl.two_pass = n_planes > 1 || coord_only || interp != GF_INTERP_BILINEAR;
    pl.n_maps = (interp > 8 && !coord_only) ? 3 : 1;
    // lean instantiation iff it is in service (GF_DISABLE_LEAN), no general-only feature is on, vector access is legal, and the
    // digital-lens flag matches the template
    const bool lean_ok = c.kernels[KV_LEAN] && (A.feat & F_GENERAL_ONLY) == 0 && (A.feat & F_LEAN_REQUIRED) == F_LEAN_REQUIRED &&
                         (((A.feat & F_DIGITAL) != 0) == (c.digital != GF_LENS_NONE));
    // packed kernel: magnitudes its fast paths assume (F_WILD clear); two-pass: the coordinate-writing variant, except for EWA whose
    // probe positions only the scalar kernels evaluate
    const KernelVariant packed = pl.two_pass ? KV_PACKED_COORDS : KV_PACKED;
    const bool packed_ok = lean_ok && c.kernels[packed] && (A.feat & F_WILD) == 0 && pl.n_maps == 1;
    pl.kernel = packed_ok ? packed : (lean_ok ? KV_LEAN : KV_GENERAL);
    // filtered pre-pass: rolling shutter on, geometry that fits the queue's entries; host tables known to be wild / IBIS take the
    // guarded path, which has no tail launch
    pl.filter = packed_ok && filter_pair(c.lens, c.digital) && (A.feat & F_RS) && !c.no_filter && A.out_cols <= WarpArgs::X2Filter::kMaxCols &&
                A.out_rows <= WarpArgs::X2Filter::kMaxRows && (tables_on_device || table_flags == 0);
    return pl;
}

// Planes of one frame that share their geometry (GBRAPF32's four R32f planes, the U and V planes of planar YUV, ...):
// every KernelParams field except plane_index and background must agree, as must buffer sizes, strides and rects.
bool planes_share_geometry(const gf_kernel_params* p, const gf_buffer_desc* in, const gf_buffer_desc* out, size_t n) {
    for (size_t i = 1; i < n; ++i) {
        gf_kernel_params a = p[0], b = p[i];
        a.plane_index = b.plane_index = 0;
        memset(a.background, 0, sizeof(a.background)); memset(b.background, 0, sizeof(b.background));
        if (memcmp(&a, &b, sizeof(a)) != 0) return false;
        const gf_buffer_desc* d[2][2] = {{&in[0], &in[i]}, {&out[0], &out[i]}};
        for (auto& q : d) {
            if (q[0]->width != q[1]->width || q[0]->height != q[1]->height || q[0]->stride != q[1]->stride || q[0]->len != q[1]->len ||
                q[0]->has_rect != q[1]->has_rect || memcmp(q[0]->rect, q[1]->rect, sizeof(q[0]->rect)) != 0 ||
                q[0]->has_rotation != q[1]->has_rotation || q[0]->rotation != q[1]->rotation || q[0]->kind != q[1]->kind) return false;
        }
    }
    return true;
}

const dim3 kBlock(GF_BLOCK_X, GF_BLOCK_Y);

// One call through the warp: the steps of run_frame and what they hand on to each other.
struct FrameRun {
    gf_cuda_ctx* const ctx; const FrameJob& job;
    std::string* const err = &ctx->last_error;
    const gf_kernel_params* const p = job.p;
    const cudaStream_t st = job.stream ? (cudaStream_t)job.stream : ctx->stream.get();
    const bool fused = job.n > 1 && ctx->fn_shade && planes_share_geometry(p, job.in, job.out, job.n);   // one coordinate pass
    const bool overlays = ctx->overlays && !fused && !job.coord_only;   // preview overlays, on every plane rendered on its own
    const bool host = std::any_of(job.in, job.in + job.n, [](const gf_buffer_desc& b) { return b.kind == GF_BUF_HOST; }) ||
                      std::any_of(job.out, job.out + job.n, [](const gf_buffer_desc& b) { return b.kind == GF_BUF_HOST; });
    std::vector<gf_buffer_desc> in{job.in, job.in + job.n}, out{job.out, job.out + job.n};   // what the kernels read and write
    bool src_private = false;               // in[0] is the context's staged copy of a HOST input
    WarpArgs T;                             // the call's tables, which every plane's arguments start from
    Slot* slot = nullptr;                   // the table slot of this call, if it uses one (host tables, or a mesh to widen)
    size_t table_rows = 0;                  // host tables: the rows copied and scanned, the most any plane reads
    uint32_t table_flags = TBL_WILD;        // host-known verdict of those rows: device tables are not trusted until validated
    const uint8_t* drawing_dev = nullptr;

    // Tables and mesh, once per call: host tables are copied through a slot and scanned on the host; a mesh is widened to f64 on the
    // device.  HOST planes: their device copies, which the planes are rendered from.
    int stage() {
        if (job.grow_staging) CK(err, ctx->plane_staging.reserve(job.n, job.in, job.out, st));
        memset(&T, 0, sizeof(T));
        if (!job.tables_on_device || job.mesh_len > 0) {      // device tables still need a slot for the widened mesh
            slot = &ctx->slots[ctx->next_slot];
            ctx->next_slot = (ctx->next_slot + 1) % kSlots;
            CK(err, cudaEventSynchronize(slot->done.get()));            // the slot's previous frame has consumed its tables
        }
        if (job.tables_on_device) {
            // the verdict travels with the data: a device word written on this stream (or ordered before it) by whoever produced the table
            T.table_flags = job.table_flags_dev ? job.table_flags_dev : ctx->const_flags.ptr + 1;
            T.matrices = job.matrices;
            T.mesh = job.mesh_len ? job.mesh : nullptr;
        } else {
            for (size_t i = 0; i < job.n; ++i) table_rows = std::max(table_rows, (size_t)p[i].matrix_count);
            const size_t mat_bytes = table_rows * GF_MATRIX_STRIDE * sizeof(float);
            memcpy(slot->h_mat.ptr, job.matrices, mat_bytes);
            table_flags = gf_table_flags_host(slot->h_mat.ptr, table_rows);
            CK(err, cudaMemcpyAsync(slot->d_mat.ptr, slot->h_mat.ptr, mat_bytes, cudaMemcpyHostToDevice, st));
            T.matrices = slot->d_mat.ptr;
            if (job.mesh_len) {
                memcpy(slot->h_mesh.ptr, job.mesh, job.mesh_len * sizeof(float));
                CK(err, cudaMemcpyAsync(slot->d_mesh.ptr, slot->h_mesh.ptr, job.mesh_len * sizeof(float), cudaMemcpyHostToDevice, st));
                T.mesh = slot->d_mesh.ptr;
            }
        }
        T.mesh_len = (int)job.mesh_len;
        if (job.mesh_len) {                                    // cpu_undistort.rs:539 — `mesh_data.iter().map(|x| *x as f64)`, once per frame
            double* const m64 = slot->d_mesh64.ptr;
            widen_mesh_kernel<<<(unsigned)((job.mesh_len + 255) / 256), 256, 0, st>>>(T.mesh, m64, (int)job.mesh_len, (float)p->width, (float)p->height);
            CK(err, cudaGetLastError());
            T.mesh64 = m64; T.mesh_aux = reinterpret_cast<const MeshAux*>(m64 + GF_MESH_MAX_LEN);
        }
        if (host) {                                            // opencl.rs:359 `self.src.write(buffer)`
            nvtxRangePushA("gf_h2d_frame");
            const int rc = ctx->plane_staging.upload(job.n, job.in, job.out, p, false, st, err, in.data(), out.data());
            nvtxRangePop();
            if (rc != GF_OK) return rc;
            src_private = job.in[0].kind == GF_BUF_HOST;
        }
        return GF_OK;
    }

    // Preview overlays, input stage: drawing entries with stage bit 0 are drawn onto the device copy of the input.
    int draw_input_overlays() {
        if (!overlays || job.n != 1) return GF_OK;
        bool any_input_stage = false;
        if ((p->flags & GF_FLAG_DRAWING_ENABLED) && job.drawing && job.drawing_len) {
            CK(err, ctx->h_drawing.reserve(job.drawing_len, st));   // (a growing reserve waits for the stream itself)
            CK(err, ctx->d_drawing.reserve(job.drawing_len, st));
            CK(err, cudaStreamSynchronize(st));                     // the previous frame's upload has left the pinned copy
            for (size_t i = 0; i < job.drawing_len; ++i) { const uint8_t d = job.drawing[i]; ctx->h_drawing.ptr[i] = d; any_input_stage |= (d != 0 && (d & 1u) == 0u); }
            CK(err, cudaMemcpyAsync(ctx->d_drawing.ptr, ctx->h_drawing.ptr, job.drawing_len, cudaMemcpyHostToDevice, st));   // opencl.rs: buf_drawing.write(drawing_buffer)
            drawing_dev = ctx->d_drawing.ptr;
        }
        if (!any_input_stage) return GF_OK;
        if (!src_private) {                                    // never draw into the caller's buffer: private copy
            CK(err, ctx->src_ovl.reserve(in[0].len, st));
            CK(err, cudaMemcpyAsync(ctx->src_ovl.ptr, in[0].ptr, in[0].len, cudaMemcpyDeviceToDevice, st));
            in[0].ptr = ctx->src_ovl.ptr;
        }
        const LayoutInfo& L = kLayouts[ctx->combo.layout];
        if (gf_internal_draw_overlays((void*)st, (uint8_t*)in[0].ptr, in[0].len, in[0].width, in[0].height, p->stride, p, L.channels, L.scalar, 1,
                                      drawing_dev, job.drawing_len) != GF_OK) return fail(err, GF_ERR_CUDA, "overlay kernel (input stage) failed");
        return GF_OK;
    }

    // The planes: one coordinate pass for all of them when they share a geometry, otherwise each plane on its own.
    int render() {
        if (fused) return render_planes(0, job.n);
        for (size_t i = 0; i < job.n; ++i) { const int rc = render_planes(i, 1); if (rc != GF_OK) return rc; }
        return GF_OK;
    }

    // Planes [first, first + count) of one geometry: uniforms, launch geometry and plan of the first, pass 1 (or the whole frame), then
    // pass 2, one sampling launch per plane.
    int render_planes(size_t first, size_t count) {
        WarpArgs A = T;
        A.p = p[first];
        A.src = (const uint8_t*)in[first].ptr; A.dst = (uint8_t*)out[first].ptr; A.src_len = in[first].len; A.dst_len = out[first].len;
        // a plane that reads fewer rows than the call staged has the verdict of its own rows
        const uint32_t flags = (size_t)A.p.matrix_count < table_rows ? gf_table_flags_host(slot->h_mat.ptr, (size_t)A.p.matrix_count) : table_flags;
        if (!job.tables_on_device) A.table_flags = ctx->const_flags.ptr + (flags ? 1 : 0);
        fill_uniforms(A, ctx->combo);
        const dim3 grid((A.out_cols + GF_BLOCK_X - 1) / GF_BLOCK_X, (A.out_rows + GF_BLOCK_Y - 1) / GF_BLOCK_Y);   // in range: validate
        const Plan plan = plan_frame(ctx->combo, A, flags, job.tables_on_device, count, job.coord_only);
        const FilterPrepass::Table* radial = nullptr;   // the lens's radial table when the frame runs the filtered pre-pass
        if (plan.filter) { const int rc = ctx->filter.table(A.p.k, st, err, &radial); if (rc != GF_OK) return rc; }
        if (plan.two_pass) {
            if (!ctx->fn_shade && !job.coord_only) return fail(err, GF_ERR_UNSUPPORTED_COMBO, "no sampling kernel for this pixel layout");
            CK(err, ctx->coords.reserve((size_t)A.out_cols * (size_t)A.out_rows * (size_t)plan.n_maps, st));
            A.coord_out = ctx->coords.ptr;
        }
        const KernelFn fn = ctx->combo.kernels[plan.kernel];
        if (plan.kernel == KV_PACKED || plan.kernel == KV_PACKED_COORDS) {
            // 32 x 4 threads (4 x 8 output rows... 32 x 8 pixels) per block measured 2 % faster than 32 x 8 threads (finer tail)
            const dim3 block2(GF_BLOCK_X, kPackedBlockY), grid2(grid.x, (A.out_rows + 2 * kPackedBlockY - 1) / (2 * kPackedBlockY));
            if (radial) { const int rc = ctx->filter.launch(fn, grid2, block2, A, *radial, st, err, ctx->launches); if (rc != GF_OK) return rc; }
            else CK(err, launch_pdl(fn, grid2, block2, A, st));
        } else {
            const size_t map_len = (size_t)A.out_cols * (size_t)A.out_rows;
            for (int mi = 0; mi < plan.n_maps; ++mi) {        // one launch, or three for EWA (pixel, x-probe, y-probe)
                if (plan.two_pass) { A.coord_out = ctx->coords.ptr + (size_t)mi * map_len; A.coord_shift = mi; }
                fn<<<grid, kBlock, 0, st>>>(A);
                CK(err, cudaGetLastError());
                if (mi > 0) ctx->launches++;
            }
        }
        CK(err, cudaGetLastError());
        ctx->launches++;
        if (!plan.two_pass || job.coord_only) return GF_OK;
        for (size_t i = first; i < first + count; ++i) {
            WarpArgs B = A;
            B.p = p[i];
            B.coord_out = nullptr; B.coord_in = ctx->coords.ptr; B.coord_maps = plan.n_maps; B.coord_shift = 0;
            B.src = (const uint8_t*)in[i].ptr; B.dst = (uint8_t*)out[i].ptr; B.src_len = in[i].len; B.dst_len = out[i].len;
            fill_uniforms(B, ctx->combo);
            ctx->fn_shade<<<grid, kBlock, 0, st>>>(B);
            CK(err, cudaGetLastError());
            ctx->launches++;
        }
        return GF_OK;
    }

    // Output-stage overlays, copy back, synchronisation.
    int finish() {
        if (slot) CK(err, cudaEventRecord(slot->done.get(), st));
        for (size_t i = 0; overlays && i < job.n; ++i) {      // output stage: stage-1 drawing entries + safe area, on the final pixels
            const LayoutInfo& L = kLayouts[ctx->combo.layout];
            if (gf_internal_draw_overlays((void*)st, (uint8_t*)out[i].ptr, out[i].len, out[i].width, out[i].height, p[i].output_stride, &p[i], L.channels,
                                          L.scalar, 0, drawing_dev, job.drawing_len) != GF_OK) return fail(err, GF_ERR_CUDA, "overlay kernel (output stage) failed");
        }
        if (!host) return GF_OK;
        nvtxRangePushA("gf_d2h_frame");                                                                              // opencl.rs:413
        const int rc = ctx->plane_staging.download(job.n, job.out, p, st, err);
        nvtxRangePop();
        if (rc != GF_OK) return rc;
        if (job.sync_host) CK(err, cudaStreamSynchronize(st));
        return GF_OK;
    }
};

// The start of every call that enqueues work for a context on `st`: after the previous call on the device (see gf_cuda_ctx::last_call).
int order_after_last_call(gf_cuda_ctx* ctx, cudaStream_t st) {
    if (ctx->last_stream && ctx->last_stream != st) CK(&ctx->last_error, cudaStreamWaitEvent(st, ctx->last_call.get(), 0));
    ctx->last_stream = st;
    return GF_OK;
}

// Every argument check of a call, before anything is enqueued: each plane's buffer kind and validate, then the checks of the call
// against the context, plane by plane.
int check_frame(gf_cuda_ctx* ctx, const FrameJob& job) {
    std::string* const err = &ctx->last_error;
    for (size_t i = 0; i < job.n; ++i) {
        if (job.kind >= 0 && (job.in[i].kind != job.kind || job.out[i].kind != job.kind)) return fail(err, GF_ERR_BAD_PARAMS, job.kind_error);
        const int rc = validate(err, job.p + i, job.in + i, job.out + i, ctx->combo.bpp());
        if (rc != GF_OK) return rc;
    }
    for (size_t i = 0; i < job.n; ++i) {
        const gf_kernel_params* p = &job.p[i];
        if (!job.matrices) return fail(err, GF_ERR_NO_DATA, "NoStabilizationData: matrices is null");
        if (p->width != ctx->width || p->height != ctx->height || p->output_width != ctx->output_width || p->output_height != ctx->output_height)
            return fail(err, GF_ERR_SIZE_MISMATCH, "SizeMismatch: KernelParams size differs from the size this context was created for");
        if (p->interpolation != ctx->interpolation)
            return fail(err, GF_ERR_UNSUPPORTED_COMBO, "interpolation differs from the one this context was created for");
        if ((size_t)p->matrix_count > job.matrix_rows) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch matrices: matrix_count > rows supplied");
        if (!job.tables_on_device && job.matrix_rows > ctx->max_rows) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch matrices");
        if (job.mesh_len > GF_MESH_MAX_LEN) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch buf_mesh_data");
        if (job.mesh_len > 0 && !job.mesh) return fail(err, GF_ERR_BAD_PARAMS, "mesh is null");
        if (job.mesh_len > 0 && job.mesh_len < 9) return fail(err, GF_ERR_BAD_PARAMS, "mesh shorter than its 9-value header (the reference would index out of bounds)");
        if (!job.grow_staging && job.in[i].kind == GF_BUF_HOST && job.in[i].len > ctx->host_in_len)
            return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch input");
        if (!job.grow_staging && job.out[i].kind == GF_BUF_HOST && job.out[i].len > ctx->host_out_len)
            return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch output");
        if (job.tables_on_device && (reinterpret_cast<uintptr_t>(job.matrices) & 7u)) return fail(err, GF_ERR_BAD_PARAMS, "device matrices must be 8-byte aligned");
    }
    return GF_OK;
}

// Every call that renders pixels (and the coordinate pass of ST maps): its checks, then its tables and HOST planes staged once, the
// planes rendered, copied back, and the call recorded in last_call.
int run_frame(gf_cuda_ctx* ctx, const FrameJob& job) {
    if (!ctx) return fail(nullptr, GF_ERR_BAD_PARAMS, "ctx is null");
    std::string* const err = &ctx->last_error;
    int rc = check_frame(ctx, job);
    if (rc != GF_OK) return rc;
    CK(err, cudaSetDevice(ctx->device));
    FrameRun F{ctx, job};
    if ((rc = order_after_last_call(ctx, F.st)) != GF_OK) return rc;
    if ((rc = F.stage()) == GF_OK && (rc = F.draw_input_overlays()) == GF_OK) {
        nvtxRangePushA("gf_warp_launch");
        if ((rc = F.render()) == GF_OK) rc = F.finish();
        nvtxRangePop();
    }
    CK(err, cudaEventRecord(ctx->last_call.get(), F.st));    // also after a failure: whatever was enqueued still uses the context
    return rc;
}

} // namespace

bool gf::warp_covers_output(const gf_kernel_params& p, const gf_buffer_desc& out, int bpp) {
    return p.output_rect[0] == 0 && p.output_rect[1] == 0 && p.output_rect[2] == out.width && p.output_rect[3] == out.height &&
           out.width == p.output_width && out.height == p.output_height && (p.flags & GF_FLAG_FILL_WITH_BACKGROUND) == 0 &&
           (size_t)out.height * (size_t)p.output_stride <= out.len + (size_t)(p.output_stride - out.width * bpp);
}

cudaError_t PlaneStaging::reserve(size_t n, const gf_buffer_desc* in, const gf_buffer_desc* out, cudaStream_t st) {
    if (in_.size() < n) { in_.resize(n); out_.resize(n); }
    for (size_t i = 0; i < n; ++i) {
        cudaError_t e = in[i].kind == GF_BUF_HOST ? in_[i].reserve(in[i].len, st) : cudaSuccess;
        if (e == cudaSuccess && out[i].kind == GF_BUF_HOST) e = out_[i].reserve(out[i].len, st);
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

int PlaneStaging::check(size_t n, const gf_buffer_desc* in, const gf_buffer_desc* out, std::string* err) const {
    for (size_t i = 0; i < n; ++i) {
        for (const gf_buffer_desc* b : {&in[i], &out[i]})
            if ((b->kind != GF_BUF_HOST && b->kind != GF_BUF_DEVICE) || !b->ptr)
                return fail(err, GF_ERR_BAD_PARAMS, "plane " + std::to_string(i) + ": unsupported buffer source");
        const size_t cap_in = i < in_.size() ? in_[i].len : 0, cap_out = i < out_.size() ? out_[i].len : 0;
        if ((in[i].kind == GF_BUF_HOST && in[i].len > cap_in) || (out[i].kind == GF_BUF_HOST && out[i].len > cap_out))
            return fail(err, GF_ERR_BUFFER_TOO_SMALL, "plane " + std::to_string(i) + ": HOST buffer longer than its staging");
    }
    return GF_OK;
}

int PlaneStaging::upload(size_t n, const gf_buffer_desc* in, const gf_buffer_desc* out, const gf_kernel_params* p, bool checksum, cudaStream_t st,
                         std::string* err, gf_buffer_desc* din, gf_buffer_desc* dout) {
    for (size_t i = 0; i < n; ++i) {
        din[i] = in[i]; dout[i] = out[i];
        if (in[i].kind == GF_BUF_HOST) {
            CK(err, cudaMemcpyAsync(in_[i].ptr, in[i].ptr, in[i].len, cudaMemcpyHostToDevice, st));
            din[i].kind = GF_BUF_DEVICE; din[i].ptr = in_[i].ptr;
        }
        if (out[i].kind == GF_BUF_HOST) {
            const int bpp = p[i].bytes_per_pixel;
            const bool padded = (size_t)p[i].output_stride != (size_t)out[i].width * (size_t)bpp;
            if (!warp_covers_output(p[i], out[i], bpp) || (checksum && padded))
                CK(err, cudaMemcpyAsync(out_[i].ptr, out[i].ptr, out[i].len, cudaMemcpyHostToDevice, st));
            dout[i].kind = GF_BUF_DEVICE; dout[i].ptr = out_[i].ptr;
        }
    }
    return GF_OK;
}

int PlaneStaging::download(size_t n, const gf_buffer_desc* out, const gf_kernel_params* p, cudaStream_t st, std::string* err) const {
    for (size_t i = 0; i < n; ++i) {
        if (out[i].kind != GF_BUF_HOST) continue;
        const size_t stride = (size_t)p[i].output_stride;
        if (warp_covers_output(p[i], out[i], p[i].bytes_per_pixel))
            CK(err, cudaMemcpy2DAsync(out[i].ptr, stride, out_[i].ptr, stride, (size_t)out[i].width * (size_t)p[i].bytes_per_pixel, (size_t)out[i].height,
                                      cudaMemcpyDeviceToHost, st));
        else
            CK(err, cudaMemcpyAsync(out[i].ptr, out_[i].ptr, out[i].len, cudaMemcpyDeviceToHost, st));
    }
    return GF_OK;
}

// Packed-kernel launches use programmatic stream serialization: the grid may be scheduled while the previous kernel on the stream
// (the frame's producer kernel, the previous frame's tail, ...) is still draining; every CTA executes griddepcontrol.wait before it
// touches memory, so the dependency itself is unchanged and only the kernel-to-kernel launch gap disappears.
cudaError_t gf::launch_pdl(KernelFn fn, dim3 g, dim3 b, const WarpArgs& args, cudaStream_t st) {
    cudaLaunchConfig_t cfg; memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = g; cfg.blockDim = b; cfg.dynamicSmemBytes = 0; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    void* kargs[1] = { (void*)&args };
    return cudaLaunchKernelExC(&cfg, (const void*)fn, kargs);
}

bool gf::lens_noop(int lens, const float* k) {
    switch (lens) {
    case GF_LENS_OPENCV_FISHEYE:
    case GF_LENS_SONY:               return k[0] == 0.0f && k[1] == 0.0f && k[2] == 0.0f && k[3] == 0.0f;
    case GF_LENS_GENERIC_POLYNOMIAL: { for (int i = 0; i < 12; ++i) if (!(k[i] == 0.0f)) return false; return true; }
    case GF_LENS_GOPRO:              return k[1] == 0.0f;
    default: return false;
    }
}

extern "C" {

GF_API int gf_cuda_device_count(void) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess) { cuda_error(e, "cudaGetDeviceCount", nullptr); return 0; }
    return n;
}

GF_API int gf_cuda_device_name(int device, char* buf, size_t buf_len) {
    if (!buf || buf_len == 0) return GF_ERR_BAD_PARAMS;
    cudaDeviceProp prop;
    CK(nullptr, cudaGetDeviceProperties(&prop, device));
    snprintf(buf, buf_len, "[CUDA] %s", prop.name);      // listed like "[OpenCL] ..." / "[wgpu] ..." (stabilization/mod.rs:399-410)
    return GF_OK;
}

GF_API int gf_cuda_supports(const gf_buffer_desc* in, const gf_buffer_desc* out) {
    if (!in || !out) return 0;
    const bool i = in->kind == GF_BUF_HOST || in->kind == GF_BUF_DEVICE;
    const bool o = out->kind == GF_BUF_HOST || out->kind == GF_BUF_DEVICE;
    return (i && o) ? 1 : 0;
}

GF_API const char* gf_cuda_version(void) { return "gyroflow-b200 0.1 (sm_90a)"; }
GF_API size_t gf_abi_struct_size(int which) {
    switch (which) {
    case 0: return sizeof(gf_kernel_params);  case 1: return sizeof(gf_buffer_desc);    case 2: return sizeof(gf_compute_params);
    case 3: return sizeof(gf_camera_stab);    case 4: return sizeof(gf_keyframe_track); case 5: return sizeof(gf_stab_config);
    case 6: return sizeof(gf_queue_config);   case 7: return sizeof(gf_lens_data);
    case 8: return sizeof(gf_mesh_f64);       case 9: return sizeof(gf_zoom_params);    case 11: return sizeof(gf_queue_plane);
    case 12: return sizeof(gf_checksum_plane); case 13: return sizeof(gf_sync_pair);    case 14: return sizeof(gf_sync_range);
    case 15: return sizeof(gf_sync_result);    default: return 0;
    }
}
GF_API const char* gf_cuda_backend_name(void) { return "CUDA"; }

GF_API int gf_lens_from_name(const char* id) {
    if (id) for (int i = 1; i < GF_LENS_COUNT; ++i) if (!strcmp(id, kLensNames[i])) return i;
    return GF_LENS_OPENCV_FISHEYE;     // DistortionModel::from_name falls back to the default model
}
GF_API const char* gf_lens_name(int lens_id) { return (lens_id >= 0 && lens_id < GF_LENS_COUNT) ? kLensNames[lens_id] : nullptr; }
GF_API int gf_pixel_bytes(int pixel_type) { const int l = pix_layout(pixel_type); return l >= 0 ? kLayouts[l].bpp : 0; }
GF_API int gf_combo_supported(int pixel_type, int distortion_model, int digital_lens, int interpolation) {
    Combo c;
    return make_combo(pixel_type, distortion_model, digital_lens, interpolation, &c) && c.kernels[KV_GENERAL] ? 1 : 0;
}

GF_API int gf_cuda_create(gf_cuda_ctx** out_ctx, int device, const gf_kernel_params* params, int pixel_type,
                          int distortion_model, int digital_lens,
                          const gf_buffer_desc* in, const gf_buffer_desc* out, size_t /* drawing_len: the drawing copies grow on demand */) {
    if (!out_ctx) return fail(nullptr, GF_ERR_BAD_PARAMS, "out_ctx is null");
    *out_ctx = nullptr;
    Combo combo;
    if (!make_combo(pixel_type, distortion_model, digital_lens, params ? params->interpolation : 0, &combo)) return fail(nullptr, GF_ERR_BAD_PARAMS, "unknown pixel type");
    { int rc = validate(nullptr, params, in, out, combo.bpp()); if (rc != GF_OK) return rc; }
    if (!combo.kernels[KV_GENERAL])
        return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "no kernel compiled for this (lens, digital lens, pixel type, interpolation)");

    std::unique_ptr<gf_cuda_ctx, Deleter<gf_cuda_destroy>> ctx(new gf_cuda_ctx());
    ctx->device = device; ctx->combo = combo; ctx->interpolation = params->interpolation;
    ctx->fn_shade = gf_shade_kernel(combo.layout);
    ctx->width = params->width; ctx->height = params->height; ctx->output_width = params->output_width; ctx->output_height = params->output_height;

    CK(nullptr, cudaSetDevice(device));
    CK(nullptr, ctx->filter.init(device));
    CK(nullptr, create_stream(ctx->stream));
    CK(nullptr, create_event(ctx->last_call));
    const cudaStream_t st = ctx->stream.get();
    // matrices: 14 * max(W, H) f32 (rows = height, or width for horizontal rolling shutter) — opencl.rs:268, wgpu.rs:260
    size_t rows = (size_t)std::max(std::max(params->width, params->height), std::max(params->output_width, params->output_height));
    rows = std::max(rows, (size_t)params->matrix_count);
    ctx->max_rows = rows;
    const uint32_t words[2] = { 0u, 1u };
    CK(nullptr, ctx->const_flags.reserve(2, st));
    CK(nullptr, cudaMemcpy(ctx->const_flags.ptr, words, sizeof(words), cudaMemcpyHostToDevice));
    CK(nullptr, ctx->vflags.reserve(1, st));
    for (Slot& sl : ctx->slots) {
        CK(nullptr, sl.h_mat.reserve(rows * GF_MATRIX_STRIDE, st));
        CK(nullptr, sl.d_mat.reserve(rows * GF_MATRIX_STRIDE, st));
        CK(nullptr, sl.h_mesh.reserve(GF_MESH_MAX_LEN, st));
        CK(nullptr, sl.d_mesh.reserve(GF_MESH_MAX_LEN, st));
        CK(nullptr, sl.d_mesh64.reserve(GF_MESH_MAX_LEN + (sizeof(MeshAux) + 7) / 8, st));
        CK(nullptr, create_event(sl.done));
    }
    ctx->host_in_len = in->kind == GF_BUF_HOST ? in->len : 0;
    ctx->host_out_len = out->kind == GF_BUF_HOST ? out->len : 0;
    CK(nullptr, ctx->plane_staging.reserve(1, in, out, st));
    *out_ctx = ctx.release();
    return GF_OK;
}

GF_API void gf_cuda_destroy(gf_cuda_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream.get());
    delete ctx;
    (void)cudaGetLastError();       // a failed teardown call must not fail the thread's next call
}

GF_API int gf_cuda_undistort_image(gf_cuda_ctx* ctx, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                   const gf_kernel_params* params, const float* matrices, size_t matrix_rows,
                                   const float* mesh, size_t mesh_len, const uint8_t* drawing, size_t drawing_len, void* cu_stream) {
    // the CPU path (the parity target) draws no overlay (cpu_undistort.rs:234-251,607,617): `drawing` is used only after
    // gf_cuda_set_overlays(ctx, 1) — then like the reference's GPU kernels (opencl_undistort.cl:121-154, overlay.cu)
    FrameJob job{1, in, out, params, matrices, matrix_rows, mesh, mesh_len, cu_stream};
    job.drawing = drawing; job.drawing_len = drawing_len;
    return run_frame(ctx, job);
}

GF_API int gf_cuda_undistort_image_dev(gf_cuda_ctx* ctx, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                       const gf_kernel_params* params, const float* matrices_dev, size_t matrix_rows,
                                       const float* mesh_dev, size_t mesh_len, void* cu_stream) {
    return gf_cuda_undistort_image_dev_flagged(ctx, in, out, params, matrices_dev, matrix_rows, mesh_dev, mesh_len, nullptr, cu_stream);
}

GF_API int gf_cuda_undistort_image_dev_flagged(gf_cuda_ctx* ctx, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                               const gf_kernel_params* params, const float* matrices_dev, size_t matrix_rows,
                                               const float* mesh_dev, size_t mesh_len, const uint32_t* table_flags_dev, void* cu_stream) {
    FrameJob job{1, in, out, params, matrices_dev, matrix_rows, mesh_dev, mesh_len, cu_stream};
    job.tables_on_device = true; job.table_flags_dev = table_flags_dev;
    return run_frame(ctx, job);
}

GF_API int gf_cuda_scan_tables_dev(const float* matrices_dev, size_t matrix_rows, uint32_t* table_flags_dev, void* cu_stream) {
    if (!matrices_dev || !table_flags_dev || matrix_rows == 0) return fail(nullptr, GF_ERR_BAD_PARAMS, "null argument");
    scan_tables_kernel<<<1, 1024, 0, (cudaStream_t)cu_stream>>>(matrices_dev, matrix_rows, table_flags_dev);
    CK(nullptr, cudaGetLastError());
    return GF_OK;
}

GF_API int gf_cuda_undistort_image_async(gf_cuda_ctx* ctx, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                         const gf_kernel_params* params, const float* matrices, size_t matrix_rows,
                                         const float* mesh, size_t mesh_len, void* cu_stream) {
    FrameJob job{1, in, out, params, matrices, matrix_rows, mesh, mesh_len, cu_stream};
    job.sync_host = false;
    return run_frame(ctx, job);
}

// ------------------------------------------------------------------------------------------
// ST maps — src/core/stmap.rs:6-146 without the EXR container: the two maps are returned as raw RGB f32 images
// (SpecificChannels::rgb of :131-135: x / width, 1 - y / height, 0).
// ------------------------------------------------------------------------------------------
__global__ void stmap_rgb_kernel(const uint2* __restrict__ coords, int w, int h, int pitch, float* __restrict__ out) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const uint2 e = coords[(size_t)y * pitch + x];
    float cx = 0.0f, cy = 0.0f;                              // `coords` starts zeroed and stays so where the closure returns None (:121-127)
    if (e.x != GF_COORD_MARK) { cx = __uint_as_float(e.x); cy = __uint_as_float(e.y); }
    float* o = out + ((size_t)y * w + x) * 3;
    o[0] = cx / (float)w; o[1] = 1.0f - (cy / (float)h); o[2] = 0.0f;
}

} // extern "C"

namespace {

// Both maps of one frame, enqueued on `st` without waiting — stmap.rs:73-116.  `cp`: stmap_params of the user's ComputeParams.  `ctx`:
// the gyro's ST-map context, at least new_w x new_h; it is set to this frame's size.
int enqueue_stmap_frame(gf_cuda_ctx* ctx, gf_cuda_gyro* g, gf_compute_params cp, int distortion_model, int digital_lens, size_t frame,
                        double timestamp_ms, int new_w, int new_h, float* dist_rgb_dev, float* undist_rgb_dev, cudaStream_t st) {
    const int width = cp.width, height = cp.height;
    cp.fov_scale = (double)fmaxf((float)new_w / (float)width, (float)new_h / (float)height);  // :75
    cp.width = new_w; cp.height = new_h; cp.output_width = new_w; cp.output_height = new_h;
    gf_kernel_params kp;
    const size_t max_rows = (size_t)std::max(new_w, new_h);
    std::vector<float> mats(max_rows * GF_MATRIX_STRIDE);
    size_t rows = 0;
    int rc = gf_frame_transform_at_timestamp(&cp, timestamp_ms, frame, &kp, mats.data(), max_rows, &rows, nullptr, nullptr);   // :79
    if (rc != GF_OK) return rc;
    kp.width = new_w; kp.height = new_h; kp.output_width = new_w; kp.output_height = new_h;   // :80-84
    kp.flags = (digital_lens != GF_LENS_NONE ? GF_FLAG_HAS_DIGITAL_LENS : 0) | (cp.readout_horizontal ? GF_FLAG_HORIZONTAL_RS : 0);
    // The closure of :88-109 is undistort_coord's row selection + rotate_and_distort and nothing else: run the warp kernel in
    // coordinate mode with the optional stages switched off (no lens-correction blend, no source-rect map: background mode 3
    // defers that map to the sampling stage, which never runs here).
    gf_kernel_params kq = kp;
    kq.lens_correction_amount = 1.0f; kq.background_mode = 3; kq.input_rotation = 0.0f;
    kq.translation2d[0] = kq.translation2d[1] = 0.0f;
    kq.interpolation = GF_INTERP_BILINEAR; kq.bytes_per_pixel = 1; kq.pix_element_count = 1;
    kq.stride = new_w; kq.output_stride = new_w;
    kq.source_rect[0] = kq.source_rect[1] = 0; kq.source_rect[2] = new_w; kq.source_rect[3] = new_h;
    kq.output_rect[0] = kq.output_rect[1] = 0; kq.output_rect[2] = new_w; kq.output_rect[3] = new_h;
    kq.max_pixel_value = 255.0f; kq.pixel_value_limit = 255.0f;
    gf_buffer_desc d; memset(&d, 0, sizeof(d));
    d.width = new_w; d.height = new_h; d.stride = new_w; d.kind = GF_BUF_DEVICE;
    d.ptr = undist_rgb_dev; d.len = (size_t)new_w * (size_t)new_h;                          // never dereferenced in coordinate mode
    ctx->width = ctx->output_width = new_w; ctx->height = ctx->output_height = new_h;
    FrameJob job{1, &d, &d, &kq, mats.data(), rows, nullptr, 0, (void*)st};                 // the table is staged through a slot
    job.coord_only = true;
    if ((rc = run_frame(ctx, job)) != GF_OK) return rc;
    const dim3 block(32, 8), grid(((unsigned)new_w + 31) / 32, ((unsigned)new_h + 7) / 8);
    stmap_rgb_kernel<<<grid, block, 0, st>>>(ctx->coords.ptr, new_w, new_h, new_w, undist_rgb_dev);
    CK(nullptr, cudaGetLastError());
    cp.width = width; cp.height = height; cp.output_width = width; cp.output_height = height;   // :111-112 (fov_scale stays)
    return gf_cuda_stmap_distort_dev(g, &cp, distortion_model, digital_lens, timestamp_ms, frame, dist_rgb_dev, st);
}

// An ST-map job of n frames whose arguments have been checked: both maps of every frame, enqueued on `st` in the gyro's coordinate-mode
// warp context.
int stmap_job(gf_cuda_gyro* g, const gf_compute_params& cp, int distortion_model, int digital_lens, const size_t* frames,
              const double* timestamps_ms, size_t n, const int32_t* new_w, const int32_t* new_h, float* const* dist_rgb_dev,
              float* const* undist_rgb_dev, cudaStream_t st) {
    int max_w = 0, max_h = 0;
    size_t max_px = 0;
    for (size_t i = 0; i < n; ++i) {
        max_w = std::max(max_w, new_w[i]); max_h = std::max(max_h, new_h[i]); max_px = std::max(max_px, (size_t)new_w[i] * (size_t)new_h[i]);
    }
    CK(nullptr, cudaSetDevice(g->device));
    if (!g->stmap_done) CK(nullptr, create_event(g->stmap_done));
    // The context is the previous job's: this stream waits for that job on the device.  A context too small or of another lens pair is
    // replaced, which waits for the previous job on the host.
    CK(nullptr, cudaStreamWaitEvent(st, g->stmap_done.get(), 0));
    if (!g->stmap_ctx || g->stmap_ctx->combo.lens != distortion_model || g->stmap_ctx->combo.digital != digital_lens ||
        g->stmap_ctx->max_rows < (size_t)std::max(max_w, max_h)) {
        CK(nullptr, cudaEventSynchronize(g->stmap_done.get()));
        g->stmap_ctx.reset();
        // LUMA8, bilinear, pass 1 only, for maps of up to max_w x max_h: a table slot of max(max_w, max_h) rows.  The buffer description
        // is for gf_cuda_create's validation, which wants a device pointer (coordinate mode never dereferences it).
        gf_kernel_params kq; memset(&kq, 0, sizeof(kq));
        kq.width = kq.output_width = kq.stride = kq.output_stride = max_w; kq.height = kq.output_height = max_h;
        kq.matrix_count = 1; kq.interpolation = GF_INTERP_BILINEAR; kq.bytes_per_pixel = 1; kq.pix_element_count = 1;
        gf_buffer_desc d; memset(&d, 0, sizeof(d));
        d.width = max_w; d.height = max_h; d.stride = max_w; d.kind = GF_BUF_DEVICE; d.ptr = undist_rgb_dev[0]; d.len = (size_t)max_w * (size_t)max_h;
        gf_cuda_ctx* raw = nullptr;
        const int rc = gf_cuda_create(&raw, g->device, &kq, GF_PIX_LUMA8, distortion_model, digital_lens, &d, &d, 0);
        if (rc != GF_OK) return rc;
        g->stmap_ctx.reset(raw);
    }
    gf_cuda_ctx* const ctx = g->stmap_ctx.get();
    CK(nullptr, ctx->coords.reserve(max_px, st));             // sized once for the largest frame (growing waits for the stream)
    int rc = GF_OK;
    for (size_t i = 0; i < n && rc == GF_OK; ++i)
        rc = enqueue_stmap_frame(ctx, g, cp, distortion_model, digital_lens, frames[i], timestamps_ms[i], new_w[i], new_h[i],
                                 dist_rgb_dev[i], undist_rgb_dev[i], st);
    CK(nullptr, cudaEventRecord(g->stmap_done.get(), st));    // also after a failure: whatever was enqueued still uses the context
    return rc;
}

} // namespace

extern "C" {

GF_API int gf_cuda_generate_stmap(gf_cuda_gyro* g, const gf_compute_params* cp_user, int distortion_model, int digital_lens,
                                  int per_frame, size_t frame, double timestamp_ms, int32_t* out_new_width, int32_t* out_new_height,
                                  float* dist_rgb_dev, size_t dist_capacity_floats, float* undist_rgb_dev, size_t undist_capacity_floats,
                                  void* cu_stream) {
    if (!g || !cp_user || !out_new_width || !out_new_height) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_generate_stmap: null argument");
    int rc = gf_cuda_stmap_sizes(g, cp_user, distortion_model, digital_lens, per_frame, &frame, &timestamp_ms, 1, out_new_width, out_new_height, cu_stream);
    if (rc != GF_OK) return rc;
    if (!dist_rgb_dev || !undist_rgb_dev) return GF_OK;                                      // size query
    const int new_w = *out_new_width, new_h = *out_new_height;
    const gf_compute_params cp = stmap_params(*cp_user, per_frame);
    if (dist_capacity_floats < (size_t)cp.width * cp.height * 3 || undist_capacity_floats < (size_t)new_w * new_h * 3)
        return fail(nullptr, GF_ERR_BUFFER_TOO_SMALL, "gf_cuda_generate_stmap: ST map output buffers too small");
    if (new_w > 16384) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_generate_stmap: undistorted width beyond the warp's 16384");
    if (!gf_combo_supported(GF_PIX_LUMA8, distortion_model, digital_lens, GF_INTERP_BILINEAR))           // the warp renders the undistort map
        return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "gf_cuda_generate_stmap: no warp kernel for this (lens, digital lens) pair");
    const cudaStream_t st = g->stream_of(cu_stream);
    if ((rc = stmap_job(g, cp, distortion_model, digital_lens, &frame, &timestamp_ms, 1, out_new_width, out_new_height, &dist_rgb_dev, &undist_rgb_dev, st)) != GF_OK)
        return rc;
    CK(nullptr, cudaStreamSynchronize(st));
    return GF_OK;
}

GF_API int gf_cuda_generate_stmaps_dev(gf_cuda_gyro* g, const gf_compute_params* cp_user, int distortion_model, int digital_lens, int per_frame,
                                       const size_t* frames, const double* timestamps_ms, size_t n,
                                       const int32_t* new_w, const int32_t* new_h, float* const* dist_rgb_dev, float* const* undist_rgb_dev,
                                       size_t dist_capacity_floats, size_t undist_capacity_floats, void* cu_stream) {
    if (!g || !cp_user) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_generate_stmaps_dev: null argument");
    if (n == 0) return GF_OK;
    if (!frames || !timestamps_ms || !new_w || !new_h || !dist_rgb_dev || !undist_rgb_dev) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_generate_stmaps_dev: null argument");
    const gf_compute_params cp = stmap_params(*cp_user, per_frame);
    if (cp.width < 4 || cp.height < 4) return fail(nullptr, GF_ERR_SIZE_TOO_SMALL, "gf_cuda_generate_stmaps_dev: SizeTooSmall");
    if (!gf_combo_supported(GF_PIX_LUMA8, distortion_model, digital_lens, GF_INTERP_BILINEAR) || !point_path_supported(distortion_model, digital_lens))
        return fail(nullptr, GF_ERR_UNSUPPORTED_COMBO, "gf_cuda_generate_stmaps_dev: no ST-map kernels for this (lens, digital lens) pair");
    // every argument is checked before the first launch
    for (size_t i = 0; i < n; ++i) {
        const std::string at = " at entry " + std::to_string(i);
        if (!dist_rgb_dev[i] || !undist_rgb_dev[i]) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_generate_stmaps_dev: null map buffer" + at);
        if (!stmap_size_ok(new_w[i], new_h[i])) return fail(nullptr, GF_ERR_SIZE_MISMATCH, "gf_cuda_generate_stmaps_dev: undistorted frame size out of range" + at);
        if (new_w[i] > 16384) return fail(nullptr, GF_ERR_BAD_PARAMS, "gf_cuda_generate_stmaps_dev: undistorted width beyond the warp's 16384" + at);
        if (dist_capacity_floats < (size_t)cp.width * cp.height * 3 || undist_capacity_floats < (size_t)new_w[i] * (size_t)new_h[i] * 3)
            return fail(nullptr, GF_ERR_BUFFER_TOO_SMALL, "gf_cuda_generate_stmaps_dev: ST map output buffers too small" + at);
    }
    return stmap_job(g, cp, distortion_model, digital_lens, frames, timestamps_ms, n, new_w, new_h, dist_rgb_dev, undist_rgb_dev,
                     g->stream_of(cu_stream));
}

GF_API int gf_cuda_undistort_planes_dev(gf_cuda_ctx* ctx, size_t n_planes, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                        const gf_kernel_params* params, const float* matrices_dev, size_t matrix_rows,
                                        const float* mesh_dev, size_t mesh_len, void* cu_stream) {
    return gf_cuda_undistort_planes_dev_flagged(ctx, n_planes, in, out, params, matrices_dev, matrix_rows, mesh_dev, mesh_len, nullptr, cu_stream);
}

GF_API int gf_cuda_undistort_planes_dev_flagged(gf_cuda_ctx* ctx, size_t n_planes, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                                const gf_kernel_params* params, const float* matrices_dev, size_t matrix_rows,
                                                const float* mesh_dev, size_t mesh_len, const uint32_t* table_flags_dev, void* cu_stream) {
    if (!ctx || !in || !out || !params || n_planes == 0) return fail(ctx ? &ctx->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    FrameJob job{n_planes, in, out, params, matrices_dev, matrix_rows, mesh_dev, mesh_len, cu_stream};
    job.kind = GF_BUF_DEVICE; job.kind_error = "gf_cuda_undistort_planes_dev takes DEVICE buffers";
    job.tables_on_device = true; job.table_flags_dev = table_flags_dev;
    return run_frame(ctx, job);
}

// The planes of one frame in HOST memory — what the render path hands over for planar software frames (rendering/mod.rs:596-629:
// every plane a BufferSource::Cpu slice): stage every plane to the device, render them like gf_cuda_undistort_planes_dev (one
// coordinate pass shared by the planes of one geometry), copy every plane back, synchronise.  Host tables, like gf_cuda_undistort_image;
// unlike it, planes of any length (the context's staging grows to them).
GF_API int gf_cuda_undistort_planes(gf_cuda_ctx* ctx, size_t n_planes, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                    const gf_kernel_params* params, const float* matrices, size_t matrix_rows,
                                    const float* mesh, size_t mesh_len, void* cu_stream) {
    if (!ctx || !in || !out || !params || n_planes == 0) return fail(ctx ? &ctx->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    FrameJob job{n_planes, in, out, params, matrices, matrix_rows, mesh, mesh_len, cu_stream};
    job.kind = GF_BUF_HOST; job.kind_error = "gf_cuda_undistort_planes takes HOST buffers (DEVICE: gf_cuda_undistort_planes_dev)";
    job.grow_staging = true;
    return run_frame(ctx, job);
}

// Host-only: which kernel variant would render this frame (no CUDA call, no context).  table_flags: 0 = validated tame tables without
// IBIS rows, non-zero = anything else.  Returns 0 general, 1 lean, 2 packed, 3 packed + trusted tables, | 0x10 two-pass (plan_frame,
// the planner run_frame uses), or a negative GF_ERR_*.  A planning aid for integrators and the hook the CPU-only tests use to check
// the host logic.  gf_cuda_plan_features also writes the frame's feature word (F_* of warp_kernel.cuh) to *feat_out: the bits
// fill_uniforms computes, plus F_FILTER when the plan runs the filtered pre-pass (FilterPrepass::launch sets that bit at launch time).
GF_API int gf_cuda_plan_features(const gf_kernel_params* params, int pixel_type, int distortion_model, int digital_lens,
                                 const gf_buffer_desc* in, const gf_buffer_desc* out, size_t mesh_len, uint32_t table_flags, size_t n_planes,
                                 uint32_t* feat_out) {
    if (feat_out) *feat_out = 0;
    if (!params || !in || !out) return GF_ERR_BAD_PARAMS;
    Combo c;
    if (!make_combo(pixel_type, distortion_model, digital_lens, params->interpolation, &c)) return GF_ERR_BAD_PARAMS;
    { int rc = validate(nullptr, params, in, out, c.bpp()); if (rc != GF_OK) return rc; }
    if (!c.kernels[KV_GENERAL]) return GF_ERR_UNSUPPORTED_COMBO;
    WarpArgs A; memset(&A, 0, sizeof(A));
    A.p = *params; A.mesh_len = (int)mesh_len;
    A.src = (const uint8_t*)in->ptr; A.dst = (uint8_t*)out->ptr; A.src_len = in->len; A.dst_len = out->len;
    fill_uniforms(A, c);
    Plan pl = plan_frame(c, A, table_flags, false, n_planes, false);
    if (pl.filter) { std::vector<float4> rows(GF_RADIAL_ROWS); pl.filter = radial_table_cap(A.p.k, rows.data()) > 0.0f; }   // as FilterPrepass::table
    // packed: the trusted path runs when the table's verdict word is 0, which the host knows only for tables it scanned
    const int v = pl.kernel == KV_GENERAL ? 0 : (pl.kernel == KV_LEAN ? 1 : (table_flags == 0 ? 3 : 2));
    if (feat_out) *feat_out = A.feat | (pl.filter ? (uint32_t)F_FILTER : 0u);
    return v | (pl.two_pass ? 0x10 : 0);
}

GF_API int gf_filter_radial_table(const float* k, float* rows_out, size_t rows_cap, float* a_cap_out) {
    if (!k || !rows_out || !a_cap_out || rows_cap < (size_t)GF_RADIAL_ROWS) return GF_ERR_BAD_PARAMS;
    std::vector<float4> rows(GF_RADIAL_ROWS);
    *a_cap_out = radial_table_cap(k, rows.data());
    memcpy(rows_out, rows.data(), rows.size() * sizeof(float4));
    return GF_RADIAL_ROWS;
}

GF_API int gf_cuda_plan(const gf_kernel_params* params, int pixel_type, int distortion_model, int digital_lens,
                        const gf_buffer_desc* in, const gf_buffer_desc* out, size_t mesh_len, uint32_t table_flags, size_t n_planes) {
    return gf_cuda_plan_features(params, pixel_type, distortion_model, digital_lens, in, out, mesh_len, table_flags, n_planes, nullptr);
}

GF_API int gf_cuda_validate_tables_dev(gf_cuda_ctx* ctx, const float* matrices_dev, size_t matrix_rows) {
    if (!ctx || !matrices_dev) return fail(ctx ? &ctx->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    std::string* const err = &ctx->last_error;
    CK(err, cudaSetDevice(ctx->device));
    // A synchronous QUERY: nothing is cached.  (Round 1 kept a pointer-keyed cache of verdicts; a table rewritten in place or an
    // allocation reused at the same address was then silently trusted.)  To render device tables on the trusted path pass a verdict
    // word to gf_cuda_undistort_image_dev_flagged — written by gf_cuda_scan_tables_dev or by gf_cuda_frame_transform_dev.
    CK(err, cudaDeviceSynchronize());                               // the table may have been written on any stream
    scan_tables_kernel<<<1, 1024, 0, ctx->stream.get()>>>(matrices_dev, matrix_rows, ctx->vflags.ptr);
    CK(err, cudaGetLastError());
    uint32_t f = 0;
    CK(err, cudaMemcpyAsync(&f, ctx->vflags.ptr, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream.get()));
    CK(err, cudaStreamSynchronize(ctx->stream.get()));
    return (int)f;      // 0 = tame and IBIS-free; bit 0 = wild entry, bit 1 = IBIS rows present (both still render correctly, on the guarded path)
}

GF_API int gf_cuda_synchronize(gf_cuda_ctx* ctx) {
    if (!ctx) return fail(nullptr, GF_ERR_BAD_PARAMS, "ctx is null");
    std::string* const err = &ctx->last_error;
    CK(err, cudaSetDevice(ctx->device));
    CK(err, cudaStreamSynchronize(ctx->stream.get()));
    if (ctx->last_stream && ctx->last_stream != ctx->stream.get()) CK(err, cudaStreamSynchronize(ctx->last_stream));   // calls made with a caller-supplied stream
    return GF_OK;
}

GF_API int gf_cuda_filter_stats(gf_cuda_ctx* ctx, uint64_t* out6) {
    if (!ctx || !out6) return fail(ctx ? &ctx->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    int rc = gf_cuda_synchronize(ctx);
    if (rc != GF_OK) return rc;
    return ctx->filter.stats(ctx->stream.get(), &ctx->last_error, out6);
}

GF_API int gf_cuda_set_overlays(gf_cuda_ctx* ctx, int enabled) {
    if (!ctx) return fail(nullptr, GF_ERR_BAD_PARAMS, "ctx is null");
    ctx->overlays = enabled ? 1 : 0;
    return GF_OK;
}

GF_API const char* gf_cuda_last_error(gf_cuda_ctx* ctx) { return ctx ? ctx->last_error.c_str() : g_last_error.c_str(); }
GF_API uint64_t gf_cuda_launch_count(gf_cuda_ctx* ctx) { return ctx ? ctx->launches : 0; }

} // extern "C"
