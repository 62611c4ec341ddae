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

namespace {

struct QSlot {
    gf_cuda_ctx* ctx = nullptr;
    cudaStream_t stream = nullptr;
    cudaEvent_t done = nullptr;
    float* d_mat = nullptr;
    uint32_t* d_flags = nullptr;
    float* h_mesh = nullptr; float* d_mesh = nullptr;      // per-frame mesh staging (pinned / device)
    uint64_t* d_sum = nullptr; uint64_t* h_sum = nullptr;  // checksum (device word, pinned host copy)
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
    gf_cuda_gyro* gyro = nullptr;
    std::vector<QSlot> slots;
    std::deque<int> fifo;                 // slots in submission order
    int next = 0;
    size_t max_rows = 0;
    unsigned long long launches = 0;
    std::string last_error;
};

namespace {
int qfail(gf_cuda_queue* q, int code, const std::string& msg) { if (q) q->last_error = msg; return code; }
int qcuda(gf_cuda_queue* q, cudaError_t e, const char* what) {
    return qfail(q, GF_ERR_CUDA, std::string(what) + ": " + cudaGetErrorName(e) + " (" + cudaGetErrorString(e) + ")");
}
#define QCK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return qcuda(q, e_, #call); } while (0)

int finish_slot(gf_cuda_queue* q, QSlot& s) {
    if (!s.busy) return GF_OK;
    QCK(cudaEventSynchronize(s.done));
    s.busy = false;
    return GF_OK;
}
} // namespace

extern "C" {

GF_API int gf_cuda_bind_thread_to_device(int device) {
    char bdf[32] = {0};
    if (cudaDeviceGetPCIBusId(bdf, sizeof(bdf), device) != cudaSuccess) { (void)cudaGetLastError(); return GF_ERR_CUDA; }
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
    if (e != cudaSuccess) { (void)cudaGetLastError(); return GF_ERR_CUDA; }
    return GF_OK;
}
GF_API int gf_cuda_host_unregister(void* ptr) {
    if (!ptr) return GF_ERR_BAD_PARAMS;
    const cudaError_t e = cudaHostUnregister(ptr);
    if (e != cudaSuccess) { (void)cudaGetLastError(); return GF_ERR_CUDA; }
    return GF_OK;
}

GF_API int gf_cuda_checksum_dev(const void* ptr_dev, size_t len, uint64_t* out_dev, void* cu_stream) {
    if (!ptr_dev || !out_dev) return GF_ERR_BAD_PARAMS;
    cudaStream_t st = (cudaStream_t)cu_stream;
    if (cudaMemsetAsync(out_dev, 0, sizeof(uint64_t), st) != cudaSuccess) { (void)cudaGetLastError(); return GF_ERR_CUDA; }
    const size_t n = len / 4;
    if (n) checksum_kernel<<<132 * 4, 256, 0, st>>>(reinterpret_cast<const uint32_t*>(ptr_dev), n, reinterpret_cast<unsigned long long*>(out_dev));
    if (cudaGetLastError() != cudaSuccess) return GF_ERR_CUDA;
    return GF_OK;
}

GF_API int gf_cuda_queue_create(gf_cuda_queue** out, const gf_queue_config* cfg, const gf_compute_params* cp,
                                const gf_buffer_desc* in_proto, const gf_buffer_desc* out_proto) {
    if (!out || !cfg || !cp || !in_proto || !out_proto) return GF_ERR_BAD_PARAMS;
    *out = nullptr;
    if (cfg->depth < 1 || cfg->depth > 16) return GF_ERR_BAD_PARAMS;
    gf_cuda_queue* q = new gf_cuda_queue();
    q->cfg = *cfg; q->cp = *cp;
    auto bail = [&](int rc) { gf_cuda_queue_destroy(q); return rc; };
    if (cudaSetDevice(cfg->device) != cudaSuccess) { (void)cudaGetLastError(); return bail(GF_ERR_CUDA); }
    if (cfg->pin_numa) (void)gf_cuda_bind_thread_to_device(cfg->device);      // before any page-locked staging is allocated
    int rc = gf_cuda_gyro_upload(&q->gyro, cfg->device, cp);
    if (rc != GF_OK) return bail(rc);
    // a template KernelParams good enough for gf_cuda_create's validation (sizes, strides, interpolation, pixel size)
    gf_kernel_params kp; memset(&kp, 0, sizeof(kp));
    kp.matrix_count = 1;
    rc = gf_get_frame_transform_at(&cfg->stab, cp, in_proto, out_proto, nullptr, 0, 0.0, 0, 1.0, &kp);
    if (rc != GF_OK) return bail(rc);
    q->max_rows = (size_t)(cp->width > cp->height ? cp->width : cp->height);
    q->slots.resize((size_t)cfg->depth);
    for (QSlot& s : q->slots) {
        rc = gf_cuda_create(&s.ctx, cfg->device, &kp, cfg->stab.pixel_type, cfg->distortion_model, cfg->digital_lens, in_proto, out_proto, 0);
        if (rc != GF_OK) { q->last_error = gf_cuda_last_error(nullptr); return bail(rc); }
        cudaError_t e;
        if ((e = cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking)) != cudaSuccess ||
            (e = cudaEventCreateWithFlags(&s.done, cudaEventDisableTiming)) != cudaSuccess ||
            (e = cudaMalloc(&s.d_mat, q->max_rows * GF_MATRIX_STRIDE * sizeof(float))) != cudaSuccess ||
            (e = cudaMalloc(&s.d_flags, sizeof(uint32_t))) != cudaSuccess ||
            (e = cudaMallocHost(&s.h_mesh, GF_MESH_MAX_LEN * sizeof(float))) != cudaSuccess ||
            (e = cudaMalloc(&s.d_mesh, GF_MESH_MAX_LEN * sizeof(float))) != cudaSuccess ||
            (e = cudaMalloc(&s.d_sum, sizeof(uint64_t))) != cudaSuccess ||
            (e = cudaMallocHost(&s.h_sum, sizeof(uint64_t))) != cudaSuccess) { qcuda(q, e, "queue slot allocation"); return bail(GF_ERR_CUDA); }
        *s.h_sum = 0;
    }
    *out = q;
    return GF_OK;
}

GF_API int gf_cuda_queue_submit(gf_cuda_queue* q, size_t frame, double timestamp_ms, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                const float* mesh, size_t mesh_len) {
    if (!q || !in || !out) return qfail(q, GF_ERR_BAD_PARAMS, "null argument");
    if (mesh_len > GF_MESH_MAX_LEN) return qfail(q, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch buf_mesh_data");
    QCK(cudaSetDevice(q->cfg.device));
    QSlot& s = q->slots[(size_t)q->next];
    if (s.busy) return qfail(q, GF_ERR_BAD_PARAMS, "queue full: gf_cuda_queue_wait for the oldest frame first");
    nvtxRangePushA("gf_queue_submit");
    // FrameTransform::at_timestamp on the device: rows x 14 table + its trust verdict, then the per-buffer half of KernelParams
    gf_kernel_params kp; size_t rows = 0; double fov = 1.0, minimal_fov = 1.0;
    int rc = gf_cuda_frame_transform_dev_flagged(q->gyro, &q->cp, timestamp_ms, frame, &kp, s.d_mat, q->max_rows, s.d_flags,
                                                 &rows, &fov, &minimal_fov, (void*)s.stream);
    if (rc != GF_OK) { nvtxRangePop(); return qfail(q, rc, "gf_cuda_frame_transform_dev_flagged failed"); }
    q->launches++;
    rc = gf_get_frame_transform_at(&q->cfg.stab, &q->cp, in, out, mesh, mesh_len, timestamp_ms, frame, minimal_fov, &kp);
    if (rc != GF_OK) { nvtxRangePop(); return qfail(q, rc, "gf_get_frame_transform_at failed"); }
    const float* mesh_dev = nullptr;
    if (mesh && mesh_len) {
        memcpy(s.h_mesh, mesh, mesh_len * sizeof(float));
        cudaError_t e = cudaMemcpyAsync(s.d_mesh, s.h_mesh, mesh_len * sizeof(float), cudaMemcpyHostToDevice, s.stream);
        if (e != cudaSuccess) { nvtxRangePop(); return qcuda(q, e, "mesh upload"); }
        mesh_dev = s.d_mesh;
    }
    const unsigned long long l0 = gf_cuda_launch_count(s.ctx);
    rc = gf_internal_run_frame(s.ctx, in, out, &kp, s.d_mat, rows, mesh_dev, mesh_dev ? mesh_len : 0, s.d_flags, (void*)s.stream,
                               q->cfg.checksum ? s.d_sum : nullptr);
    if (rc != GF_OK) { q->last_error = gf_cuda_last_error(s.ctx); nvtxRangePop(); return rc; }
    q->launches += gf_cuda_launch_count(s.ctx) - l0 + (q->cfg.checksum ? 1 : 0);
    if (q->cfg.checksum) {
        cudaError_t e = cudaMemcpyAsync(s.h_sum, s.d_sum, sizeof(uint64_t), cudaMemcpyDeviceToHost, s.stream);
        if (e != cudaSuccess) { nvtxRangePop(); return qcuda(q, e, "checksum download"); }
    }
    cudaError_t e = cudaEventRecord(s.done, s.stream);
    nvtxRangePop();
    if (e != cudaSuccess) return qcuda(q, e, "cudaEventRecord");
    s.busy = true; s.frame = frame;
    q->fifo.push_back(q->next);
    q->next = (q->next + 1) % (int)q->slots.size();
    return GF_OK;
}

GF_API int gf_cuda_queue_wait(gf_cuda_queue* q, size_t* out_frame, uint64_t* out_checksum) {
    if (!q) return GF_ERR_BAD_PARAMS;
    if (q->fifo.empty()) return qfail(q, GF_ERR_NO_DATA, "nothing in flight");
    QSlot& s = q->slots[(size_t)q->fifo.front()];
    q->fifo.pop_front();
    int rc = finish_slot(q, s);
    if (rc != GF_OK) return rc;
    if (out_frame) *out_frame = s.frame;
    if (out_checksum) *out_checksum = *s.h_sum;
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
    for (QSlot& s : q->slots) {
        if (s.stream) cudaStreamSynchronize(s.stream);
        if (s.ctx) gf_cuda_destroy(s.ctx);
        if (s.d_mat) cudaFree(s.d_mat);
        if (s.d_flags) cudaFree(s.d_flags);
        if (s.h_mesh) cudaFreeHost(s.h_mesh);
        if (s.d_mesh) cudaFree(s.d_mesh);
        if (s.d_sum) cudaFree(s.d_sum);
        if (s.h_sum) cudaFreeHost(s.h_sum);
        if (s.done) cudaEventDestroy(s.done);
        if (s.stream) cudaStreamDestroy(s.stream);
    }
    if (q->gyro) gf_cuda_gyro_free(q->gyro);
    (void)cudaGetLastError();
    delete q;
}

} // extern "C"
