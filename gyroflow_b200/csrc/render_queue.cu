// render_queue.cu — the frame-sharded render queue of one GPU (SURVEY §8e, §7.9).
//
// What the reference does per frame on the render path (rendering/mod.rs:451,531-542,657-661): the ffmpeg frame callback calls
// `Stabilization::get_frame_transform_at` (FrameTransform::at_timestamp + the per-buffer fields) and then `process_pixels`,
// strictly one frame after another on one device; `render_queue.rs:550-612` only runs whole jobs side by side.  Frames are
// independent units (at_timestamp depends on immutable ComputeParams + the timestamp, frame_transform.rs:165), so this queue keeps
// `depth` of them in flight on one GPU and lets a box shard `i -> GPU (i mod G)` across processes with no data-path collective.
//
// One slot = one stream + one warp context (its own device staging when the buffers are HOST) + a device matrix table with its
// trust verdict word.  Per submitted frame, all enqueued on the slot's stream, nothing synchronous:
//     producer kernel (gf_cuda_frame_transform_dev_flagged: table + verdict)  ->  [mesh H2D]  ->  [frame H2D]  ->  warp kernel
//     ->  [checksum kernel]  ->  [frame D2H]  ->  event
// Slots are used round-robin; submit() waits for a slot's previous frame only when it comes round again, wait() hands finished
// frames back in submission order (output order restored by frame index on the host, as §8e asks).
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <sched.h>
#include <cstdio>
#include <cstring>
#include <cstdlib>
#include <string>
#include <vector>
#include <deque>
#include "../../include/gyroflow_cuda.h"
#include "c_abi_internal.h"

using namespace gf;

namespace {

struct QSlot {
    std::unique_ptr<gf_cuda_ctx, Deleter<gf_cuda_destroy>> ctx;
    Stream stream;
    Event done;
    GrowBuf<float> d_mat;
    GrowBuf<uint32_t> d_flags;
    GrowBuf<float, true> h_mesh; GrowBuf<float> d_mesh;      // per-frame mesh staging (pinned / device)
    GrowBuf<uint64_t> d_sum; GrowBuf<uint64_t, true> h_sum;  // checksum (device word, pinned host copy)
    bool busy = false;
    size_t frame = 0;
};

// sum(word[i] * (2 i + 1)) mod 2^64: order-independent, so blocks may add their partial sums in any order
__global__ void checksum_kernel(const uint32_t* __restrict__ w, size_t n, unsigned long long* __restrict__ out) {
    unsigned long long s = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        s += (unsigned long long)w[i] * (2ull * (unsigned long long)i + 1ull);
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31u) == 0u && s) atomicAdd(out, s);
}

} // namespace

struct gf_cuda_queue {
    gf_queue_config cfg;
    gf_compute_params cp;                 // shallow copy: the arrays it points to stay owned by the caller for the queue's lifetime
    std::unique_ptr<gf_cuda_gyro, Deleter<gf_cuda_gyro_free>> gyro;
    std::vector<QSlot> slots;
    std::deque<int> fifo;                 // slots in submission order
    int next = 0;
    size_t max_rows = 0;
    unsigned long long launches = 0;
    std::string last_error;
};

namespace {
int finish_slot(gf_cuda_queue* q, QSlot& s) {
    if (!s.busy) return GF_OK;
    CK(&q->last_error, cudaEventSynchronize(s.done.get()));
    s.busy = false;
    return GF_OK;
}
} // namespace

extern "C" {

GF_API int gf_cuda_bind_thread_to_device(int device) {
    char bdf[32] = {0};
    CK(nullptr, cudaDeviceGetPCIBusId(bdf, sizeof(bdf), device));
    for (char* c = bdf; *c; ++c) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');      // sysfs uses lower-case hex
    char path[128];
    snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/local_cpulist", bdf);
    FILE* f = fopen(path, "r");
    if (!f) return 0;
    char line[1024] = {0};
    const bool got = fgets(line, sizeof(line), f) != nullptr;
    fclose(f);
    if (!got) return 0;
    cpu_set_t want, have;
    CPU_ZERO(&want);
    int n = 0;
    for (char* tok = strtok(line, ",\n"); tok; tok = strtok(nullptr, ",\n")) {                  // "32-63,96-127"
        int a = 0, b = 0;
        const int k = sscanf(tok, "%d-%d", &a, &b);
        if (k == 1) b = a;
        if (k < 1 || a < 0 || b < a) continue;
        for (int c = a; c <= b && c < CPU_SETSIZE; ++c) CPU_SET(c, &want);
    }
    // stay inside what the process is allowed to use (cgroup / taskset): intersect, and keep the old mask if the intersection is empty
    if (sched_getaffinity(0, sizeof(have), &have) == 0) {
        cpu_set_t both; CPU_AND(&both, &want, &have);
        if (CPU_COUNT(&both) == 0) return 0;
        want = both;
    }
    n = CPU_COUNT(&want);
    if (n == 0) return 0;
    if (sched_setaffinity(0, sizeof(want), &want) != 0) return GF_ERR_BAD_PARAMS;
    return n;
}

// Page-lock an existing host allocation (the decoder's frame pool, a long-lived Vec<u8>) so that HOST-buffer calls copy at the link's rate
// instead of through the driver's bounce buffers (bench: 742 vs 262 sequential 4K frames/s).  Thin wrappers over cudaHostRegister /
// cudaHostUnregister: the caller owns the lifetime — unregister before the memory is freed.
GF_API int gf_cuda_host_register(void* ptr, size_t len) {
    if (!ptr || !len) return GF_ERR_BAD_PARAMS;
    const cudaError_t e = cudaHostRegister(ptr, len, cudaHostRegisterPortable);
    if (e == cudaErrorHostMemoryAlreadyRegistered) { (void)cudaGetLastError(); return GF_OK; }
    return e == cudaSuccess ? GF_OK : cuda_error(e, "cudaHostRegister", nullptr);
}
GF_API int gf_cuda_host_unregister(void* ptr) {
    if (!ptr) return GF_ERR_BAD_PARAMS;
    CK(nullptr, cudaHostUnregister(ptr));
    return GF_OK;
}

GF_API int gf_cuda_checksum_dev(const void* ptr_dev, size_t len, uint64_t* out_dev, void* cu_stream) {
    if (!ptr_dev || !out_dev) return GF_ERR_BAD_PARAMS;
    cudaStream_t st = (cudaStream_t)cu_stream;
    CK(nullptr, cudaMemsetAsync(out_dev, 0, sizeof(uint64_t), st));
    const size_t n = len / 4;
    if (n) checksum_kernel<<<132 * 4, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(ptr_dev), n, reinterpret_cast<unsigned long long*>(out_dev));
    CK(nullptr, cudaGetLastError());
    return GF_OK;
}

GF_API int gf_cuda_queue_create(gf_cuda_queue** out, const gf_queue_config* cfg, const gf_compute_params* cp,
                                const gf_buffer_desc* in_proto, const gf_buffer_desc* out_proto) {
    if (!out || !cfg || !cp || !in_proto || !out_proto) return GF_ERR_BAD_PARAMS;
    *out = nullptr;
    if (cfg->depth < 1 || cfg->depth > 16) return GF_ERR_BAD_PARAMS;
    std::unique_ptr<gf_cuda_queue, Deleter<gf_cuda_queue_destroy>> q(new gf_cuda_queue());
    q->cfg = *cfg; q->cp = *cp;
    CK(nullptr, cudaSetDevice(cfg->device));
    if (cfg->pin_numa) (void)gf_cuda_bind_thread_to_device(cfg->device);      // before any page-locked staging is allocated
    gf_cuda_gyro* gyro = nullptr;
    int rc = gf_cuda_gyro_upload(&gyro, cfg->device, cp);
    if (rc != GF_OK) return rc;
    q->gyro.reset(gyro);
    // a template KernelParams good enough for gf_cuda_create's validation (sizes, strides, interpolation, pixel size)
    gf_kernel_params kp; memset(&kp, 0, sizeof(kp));
    kp.matrix_count = 1;
    rc = gf_get_frame_transform_at(&cfg->stab, cp, in_proto, out_proto, nullptr, 0, 0.0, 0, 1.0, &kp);
    if (rc != GF_OK) return rc;
    q->max_rows = (size_t)(cp->width > cp->height ? cp->width : cp->height);
    q->slots.resize((size_t)cfg->depth);
    for (QSlot& s : q->slots) {
        gf_cuda_ctx* ctx = nullptr;
        rc = gf_cuda_create(&ctx, cfg->device, &kp, cfg->stab.pixel_type, cfg->distortion_model, cfg->digital_lens, in_proto, out_proto, 0);
        if (rc != GF_OK) return rc;
        s.ctx.reset(ctx);
        CK(nullptr, create_stream(s.stream));
        CK(nullptr, create_event(s.done));
        const cudaStream_t st = s.stream.get();
        CK(nullptr, s.d_mat.reserve(q->max_rows * GF_MATRIX_STRIDE, st));
        CK(nullptr, s.d_flags.reserve(1, st));
        CK(nullptr, s.h_mesh.reserve(GF_MESH_MAX_LEN, st));
        CK(nullptr, s.d_mesh.reserve(GF_MESH_MAX_LEN, st));
        CK(nullptr, s.d_sum.reserve(1, st));
        CK(nullptr, s.h_sum.reserve(1, st));
        *s.h_sum.ptr = 0;
    }
    *out = q.release();
    return GF_OK;
}

GF_API int gf_cuda_queue_submit(gf_cuda_queue* q, size_t frame, double timestamp_ms, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                const float* mesh, size_t mesh_len) {
    if (!q || !in || !out) return fail(q ? &q->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    std::string* const err = &q->last_error;
    if (mesh_len > GF_MESH_MAX_LEN) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch buf_mesh_data");
    CK(err, cudaSetDevice(q->cfg.device));
    QSlot& s = q->slots[(size_t)q->next];
    if (s.busy) return fail(err, GF_ERR_BAD_PARAMS, "queue full: gf_cuda_queue_wait for the oldest frame first");
    const cudaStream_t st = s.stream.get();
    nvtxRangePushA("gf_queue_submit");
    // FrameTransform::at_timestamp on the device: rows x 14 table + its trust verdict, then the per-buffer half of KernelParams
    gf_kernel_params kp; size_t rows = 0; double fov = 1.0, minimal_fov = 1.0;
    int rc = gf_cuda_frame_transform_dev_flagged(q->gyro.get(), &q->cp, timestamp_ms, frame, &kp, s.d_mat.ptr, q->max_rows, s.d_flags.ptr,
                                                 &rows, &fov, &minimal_fov, (void*)st);
    if (rc != GF_OK) { nvtxRangePop(); return fail(err, rc, "gf_cuda_frame_transform_dev_flagged failed"); }
    q->launches++;
    rc = gf_get_frame_transform_at(&q->cfg.stab, &q->cp, in, out, mesh, mesh_len, timestamp_ms, frame, minimal_fov, &kp);
    if (rc != GF_OK) { nvtxRangePop(); return fail(err, rc, "gf_get_frame_transform_at failed"); }
    const float* mesh_dev = nullptr;
    if (mesh && mesh_len) {
        memcpy(s.h_mesh.ptr, mesh, mesh_len * sizeof(float));
        cudaError_t e = cudaMemcpyAsync(s.d_mesh.ptr, s.h_mesh.ptr, mesh_len * sizeof(float), cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) { nvtxRangePop(); return cuda_error(e, "mesh upload", err); }
        mesh_dev = s.d_mesh.ptr;
    }
    const unsigned long long l0 = gf_cuda_launch_count(s.ctx.get());
    rc = gf_internal_run_frame(s.ctx.get(), in, out, &kp, s.d_mat.ptr, rows, mesh_dev, mesh_dev ? mesh_len : 0, s.d_flags.ptr, (void*)st,
                               q->cfg.checksum ? s.d_sum.ptr : nullptr);
    if (rc != GF_OK) { q->last_error = gf_cuda_last_error(s.ctx.get()); nvtxRangePop(); return rc; }
    q->launches += gf_cuda_launch_count(s.ctx.get()) - l0 + (q->cfg.checksum ? 1 : 0);
    if (q->cfg.checksum) {
        cudaError_t e = cudaMemcpyAsync(s.h_sum.ptr, s.d_sum.ptr, sizeof(uint64_t), cudaMemcpyDeviceToHost, st);
        if (e != cudaSuccess) { nvtxRangePop(); return cuda_error(e, "checksum download", err); }
    }
    cudaError_t e = cudaEventRecord(s.done.get(), st);
    nvtxRangePop();
    if (e != cudaSuccess) return cuda_error(e, "cudaEventRecord", err);
    s.busy = true; s.frame = frame;
    q->fifo.push_back(q->next);
    q->next = (q->next + 1) % (int)q->slots.size();
    return GF_OK;
}

GF_API int gf_cuda_queue_wait(gf_cuda_queue* q, size_t* out_frame, uint64_t* out_checksum) {
    if (!q) return GF_ERR_BAD_PARAMS;
    if (q->fifo.empty()) return fail(&q->last_error, GF_ERR_NO_DATA, "nothing in flight");
    QSlot& s = q->slots[(size_t)q->fifo.front()];
    q->fifo.pop_front();
    int rc = finish_slot(q, s);
    if (rc != GF_OK) return rc;
    if (out_frame) *out_frame = s.frame;
    if (out_checksum) *out_checksum = *s.h_sum.ptr;
    return GF_OK;
}

GF_API int gf_cuda_queue_drain(gf_cuda_queue* q) {
    if (!q) return GF_ERR_BAD_PARAMS;
    while (!q->fifo.empty()) { int rc = gf_cuda_queue_wait(q, nullptr, nullptr); if (rc != GF_OK) return rc; }
    return GF_OK;
}

GF_API uint64_t gf_cuda_queue_launches(gf_cuda_queue* q) { return q ? q->launches : 0; }
GF_API const char* gf_cuda_queue_last_error(gf_cuda_queue* q) { return q ? q->last_error.c_str() : ""; }

GF_API void gf_cuda_queue_destroy(gf_cuda_queue* q) {
    if (!q) return;
    cudaSetDevice(q->cfg.device);
    for (QSlot& s : q->slots) if (s.stream) cudaStreamSynchronize(s.stream.get());
    delete q;
    (void)cudaGetLastError();       // a failed teardown call must not fail the thread's next call
}

} // extern "C"
