// c_abi_internal.h — entry points shared between the translation units of libgyroflow_cuda.so, NOT exported
// (the library is built with -fvisibility=hidden; only GF_API symbols leave it).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>
#include "../../include/gyroflow_cuda.h"
#include "frame_geometry.cuh"

namespace gf {

// ---- Errors: every entry point reports a failure through these ----

// The calling thread's last error message (gf_cuda_last_error(NULL)).
inline thread_local std::string g_last_error;

// `msg` becomes the thread's last error and, when `sink` is given, the message of the context or queue the failure belongs to.
inline int fail(std::string* sink, int code, const std::string& msg) {
    g_last_error = msg;
    if (sink) *sink = msg;
    return code;
}
// A failed CUDA call: clears the runtime's pending error, so that the thread's next call does not fail on it, and reports
// "what: name (description)".
inline int cuda_error(cudaError_t e, const char* what, std::string* sink) {
    (void)cudaGetLastError();
    return fail(sink, GF_ERR_CUDA, std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")");
}
#define CK(sink, call) do { const cudaError_t e_ = (call); if (e_ != cudaSuccess) return gf::cuda_error(e_, #call, sink); } while (0)

// ---- Owners: each CUDA resource is released by the object that holds it ----
// The objects the entry points hand out (contexts, queues, gyro uploads) are torn down by setting their device, synchronising their
// streams and deleting them: the members' destructors must not free what queued work may still use.

// A device buffer (PINNED: page-locked host memory) of `len` elements that grows on demand.  Growing waits for the stream, whose queued
// work may still use the old buffer, frees it and allocates the new size; on an empty buffer reserve is a plain allocation.
template <class T, bool PINNED = false> struct GrowBuf {
    T* ptr = nullptr; size_t len = 0;
    GrowBuf() = default;
    GrowBuf(GrowBuf&& o) noexcept : ptr(o.ptr), len(o.len) { o.ptr = nullptr; o.len = 0; }
    ~GrowBuf() { release(); }
    cudaError_t reserve(size_t n, cudaStream_t st) {
        if (n <= len) return cudaSuccess;
        if (ptr) { const cudaError_t e = cudaStreamSynchronize(st); if (e != cudaSuccess) return e; release(); }
        const cudaError_t e = PINNED ? cudaMallocHost((void**)&ptr, n * sizeof(T)) : cudaMalloc((void**)&ptr, n * sizeof(T));
        if (e == cudaSuccess) len = n; else ptr = nullptr;
        return e;
    }
private:
    void release() { if (ptr) { if (PINNED) cudaFreeHost(ptr); else cudaFree(ptr); } ptr = nullptr; len = 0; }
};

// unique_ptr deleter calling `Destroy` (cudaStreamDestroy, gf_cuda_destroy, ...)
template <auto Destroy> struct Deleter { template <class T> void operator()(T* h) const { Destroy(h); } };
using Stream = std::unique_ptr<CUstream_st, Deleter<cudaStreamDestroy>>;
using Event = std::unique_ptr<CUevent_st, Deleter<cudaEventDestroy>>;
inline cudaError_t create_stream(Stream& s) {
    cudaStream_t h = nullptr;
    const cudaError_t e = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking);
    if (e == cudaSuccess) s.reset(h);
    return e;
}
inline cudaError_t create_event(Event& ev) {
    cudaEvent_t h = nullptr;
    const cudaError_t e = cudaEventCreateWithFlags(&h, cudaEventDisableTiming);
    if (e == cudaSuccess) ev.reset(h);
    return e;
}

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

// The host half of the per-frame geometry (frame_transform.cu), shared by the matrix producer (at_timestamp) and the point path
// (at_timestamp_for_points).
// `params.keyframes.value_at_video_timestamp(typ, ts).unwrap_or(dflt)`
double keyframed(const gf_compute_params* cp, int typ, double timestamp_ms, double dflt);
// get_fov (frame_transform.rs:52-58) without its last line, `fov *= width / output_width.max(1)`, which the callers apply: the producer in
// that order, the point path as (fov * width) / output_width, like the oracle's transcription of at_timestamp_for_points.
double fov_unscaled(const gf_compute_params* cp, size_t frame, bool use_fovs, double timestamp_ms, bool for_ui);
// get_new_k — frame_transform.rs:37-51
void get_new_k(const gf_compute_params* cp, const double* camera_matrix, double fov, double (&new_k)[9]);
// Readout timing and base rotation of one frame — frame_transform.rs:221-225,243-244 (at_timestamp), :376-388 (at_timestamp_for_points)
struct FrameTiming {
    double frame_readout_time;            // get_frame_readout_time(can_invert): signed and scaled
    double row_readout_time, start_ts;    // start_ts includes the frame's per_frame_time_offsets entry
    Quat q0;                              // smoothed(ts) * org(ts)^-1 through the host tracks and sync offsets
};
FrameTiming frame_timing(const gf_compute_params* cp, size_t frame, double timestamp_ms, bool can_invert);
// camera_stab[frame] with `splines` as its spline points; absent when the frame has no entry or `splines` is null
CameraStab camera_stab_at(const gf_compute_params* cp, size_t frame, bool framebuffer_inverted, const StabSplines* splines);
// the lens model is the identity for these coefficients (c_abi.cu)
bool lens_noop(int lens, const float* k);
// the point path (zoom_kernel.cu) compiles this (lens, digital lens) pair
bool point_path_supported(int lens, int digital);

// ---- Filtered rolling-shutter pre-pass of the packed fisheye kernel (filter_prepass.cu) ----
struct WarpArgs;
typedef void (*KernelFn)(const WarpArgs);      // as kernel_registry.h
cudaError_t launch_pdl(KernelFn fn, dim3 g, dim3 b, const WarpArgs& args, cudaStream_t st);    // c_abi.cu
// The radial table (GF_RADIAL_ROWS rows, Lens2<opencv_fisheye>::approx_v) of fisheye coefficients k[0..3]: returns the conditioning cap
// on r^2 rounded down to a row boundary (NaN rows from there on), or 0 when the lens runs without the filter.
float radial_table_cap(const float* k, float4* rows);
// One per context: the radial tables of the last four lenses, the deferred-pair queue with its two ping-pong counters, and the launches
// of a filtered frame.  They rely on the context's calls being ordered on the device (gf_cuda_ctx::last_call).
class FilterPrepass {
public:
    struct Table {                             // rebuilt only once `done` has passed: it is recorded after the upload and every reader
        uint32_t key[4] = {};
        float a_cap = 0.0f;                    // radial_table_cap
        unsigned long long last_use = 0;       // 0: empty
        GrowBuf<float4, true> h; GrowBuf<float4> d; Event done;
    };
    cudaError_t init(int device) { return cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, device); }
    // The lens's table, cached by the bits of k[0..3] or built in the least recently used entry and uploaded on `st`; nullptr: no filter.
    int table(const float* k, cudaStream_t st, std::string* err, const Table** out);
    // The main launch, which defers the pairs it cannot certify, and the tail launch, which renders them; the tail is added to `launches`.
    int launch(KernelFn fn, dim3 grid, dim3 block, WarpArgs& A, const Table& t, cudaStream_t st, std::string* err, unsigned long long& launches);
    int stats(cudaStream_t st, std::string* err, uint64_t* out6) const;    // gf_cuda_filter_stats, once `st` has every frame behind it
private:
    Table tables[4];
    GrowBuf<uint32_t> queue; GrowBuf<unsigned> counts;
    unsigned long long frames = 0, uses = 0, builds = 0;
    int sm_count = 1;
};

// ---- HOST image buffers (c_abi.cu) ----
// The warp of `p` writes every pixel of `out` (output_rect = buffer = output size, no fill-with-background: the bounds test of
// cpu_undistort.rs:551 passes everywhere), and the buffer lacks at most the last row's padding.  Otherwise the pixels the warp leaves
// alone keep their previous content, like on the CPU path, so a staged output is uploaded first.
bool warp_covers_output(const gf_kernel_params& p, const gf_buffer_desc& out, int bpp);
// Device copies of a frame's HOST planes (render-queue slots, warp contexts); a DEVICE buffer is used in place.
class PlaneStaging {
public:
    cudaError_t reserve(size_t n, const gf_buffer_desc* in, const gf_buffer_desc* out, cudaStream_t st);   // growing waits for `st`
    // GF_ERR_BAD_PARAMS for a buffer of neither kind or without a pointer, GF_ERR_BUFFER_TOO_SMALL for a HOST one beyond the capacity
    int check(size_t n, const gf_buffer_desc* in, const gf_buffer_desc* out, std::string* err) const;
    // din / dout: what the warp of p[i] reads and writes.  The output is uploaded unless the warp writes every byte of it that is read
    // afterwards (covered, and no stride padding when `checksum` reads the device rows); a covered one comes back as its pixel rows.
    int upload(size_t n, const gf_buffer_desc* in, const gf_buffer_desc* out, const gf_kernel_params* p, bool checksum, cudaStream_t st,
               std::string* err, gf_buffer_desc* din, gf_buffer_desc* dout);
    int download(size_t n, const gf_buffer_desc* out, const gf_kernel_params* p, cudaStream_t st, std::string* err) const;
private:
    std::vector<GrowBuf<uint8_t>> in_, out_;
};

// What generate_stmaps does to the user's ComputeParams before either map (stmap.rs:24-35, :44-46): rotation suppressed, fovs cleared,
// no readout time unless per_frame, fov_scale 1 and the output size the frame size.
inline gf_compute_params stmap_params(const gf_compute_params& user, int per_frame) {
    gf_compute_params cp = user;
    if (!per_frame) cp.frame_readout_time = 0.0;
    cp.suppress_rotation = 1; cp.fovs = nullptr; cp.n_fovs = 0; cp.minimal_fovs = nullptr; cp.n_minimal_fovs = 0;
    cp.fov_scale = 1.0; cp.output_width = cp.width; cp.output_height = cp.height;
    return cp;
}
// The undistorted sizes gf_cuda_generate_stmap accepts (the warp that renders the undistort map takes widths up to 16384 besides)
inline bool stmap_size_ok(int w, int h) { return w >= 4 && h >= 4 && w <= 32768 && h <= 32768; }

} // namespace gf

// Preview overlays (overlay.cu): draw_pixel + draw_safe_area of opencl_undistort.cl:109-154 as a pass over a DEVICE buffer.
// count / scalar: channels and scalar kind (0 u8, 1 u16, 2 f32, 3 f16) of the pixel type.
int gf_internal_draw_overlays(void* cu_stream, uint8_t* buf_dev, size_t len, int width, int height, int stride, const gf_kernel_params* p,
                              int count, int scalar, int is_input, const uint8_t* drawing_dev, size_t drawing_len);
