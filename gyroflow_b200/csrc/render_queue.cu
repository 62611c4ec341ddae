// render_queue.cu — the frame-sharded render queue of one GPU (SURVEY §8e, §7.9).
//
// What the reference does per frame on the render path (rendering/mod.rs:451,531-542,657-661): the ffmpeg frame callback calls
// `Stabilization::get_frame_transform_at` (FrameTransform::at_timestamp + the per-buffer fields) and then `process_pixels`,
// strictly one frame after another on one device; `render_queue.rs:550-612` only runs whole jobs side by side.  Frames are
// independent units (at_timestamp depends on immutable ComputeParams + the timestamp, frame_transform.rs:165), so this queue keeps
// `depth` of them in flight on one GPU and lets a box shard `i -> GPU (i mod G)` across processes with no data-path collective.
//
// Every queue renders frames of a plane layout: 1-4 planes (a decoder frame, create_planes_proc!, rendering/mod.rs:483-651), or the
// one plane of a gf_cuda_queue_create queue.  Every plane's Stabilization has the frame's size and ComputeParams, so one producer launch
// serves all planes; per plane only the per-buffer half of KernelParams differs.  Planes of one pixel type and size fraction form a
// group, which has one warp context in each slot.
// One slot = one stream + a warp context per group + device staging of the HOST planes + a device matrix table with its trust verdict
// word.  Per submitted frame, all enqueued on the slot's stream, nothing synchronous:
//     producer kernel (gf_cuda_frame_transform_dev_flagged: table + verdict)  ->  [mesh H2D]  ->  [H2D of the HOST planes]
//     ->  one gf_cuda_undistort_planes_dev_flagged per group  ->  [one checksum launch over all planes]  ->  [D2H of the HOST planes]  ->  event
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
#include <algorithm>
#include "../../include/gyroflow_cuda.h"
#include "c_abi_internal.h"

using namespace gf;

namespace {

struct QSlot {
    Stream stream;
    Event done;
    GrowBuf<float> d_mat;
    GrowBuf<uint32_t> d_flags;
    GrowBuf<float, true> h_mesh; GrowBuf<float> d_mesh;      // per-frame mesh staging (pinned / device)
    GrowBuf<uint64_t> d_sum; GrowBuf<uint64_t, true> h_sum;  // checksum (device word, pinned host copy)
    bool busy = false;
    size_t frame = 0;
    std::vector<std::unique_ptr<gf_cuda_ctx, Deleter<gf_cuda_destroy>>> group_ctx;   // one warp context per plane group
    PlaneStaging staging;                                    // device copies of the HOST planes, sized from the prototypes
};

// sum(word[i] * (2 i + 1)) mod 2^64 over the rows of up to four descriptors read as one byte string (gf_cuda_checksum_planes_dev):
// order-independent, so blocks may add their partial sums in any order.  A block takes whole rows;
// its threads take the string's 32-bit words that the row touches.  A word cut by a row boundary gets its bytes from both rows, each
// row adding its own bytes times the word's weight, which sums to the whole word's term.
struct ChecksumRows {
    const uint8_t* ptr[4];
    unsigned long long row_bytes[4], stride[4];
    unsigned long long first_row[5];       // rows of the descriptors before k (first_row[n]: all rows)
    unsigned long long first_byte[4];      // string offset of descriptor k's first byte
    unsigned long long end;                // bytes summed: 4 * (string length / 4)
    int n;
};
__global__ void checksum_rows_kernel(const ChecksumRows P, unsigned long long* __restrict__ out) {
    unsigned long long s = 0;
    for (unsigned long long r = blockIdx.x; r < P.first_row[P.n]; r += gridDim.x) {
        int k = 0;
        while (k + 1 < P.n && r >= P.first_row[k + 1]) ++k;
        const unsigned long long lr = r - P.first_row[k];
        const uint8_t* const row = P.ptr[k] + lr * P.stride[k];
        const unsigned long long g0 = P.first_byte[k] + lr * P.row_bytes[k];                 // string offset of the row's first byte
        const unsigned long long g1 = min(g0 + P.row_bytes[k], P.end);                       // past its last summed byte
        if (g0 >= g1) continue;
        for (unsigned long long w = (g0 >> 2) + threadIdx.x; w < ((g1 + 3) >> 2); w += blockDim.x) {
            const unsigned long long b0 = max(4ull * w, g0), b1 = min(4ull * w + 4ull, g1);
            uint32_t v = 0;
            if (b0 == 4ull * w && b1 == b0 + 4ull && (reinterpret_cast<uintptr_t>(row + (b0 - g0)) & 3u) == 0u) {
                v = *reinterpret_cast<const uint32_t*>(row + (b0 - g0));
            } else {
                for (unsigned long long b = b0; b < b1; ++b) v |= (uint32_t)row[b - g0] << (8u * (unsigned)(b - 4ull * w));
            }
            s += (unsigned long long)v * (2ull * w + 1ull);
        }
    }
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31u) == 0u && s) atomicAdd(out, s);
}

// One plane of the queue's layout.
struct QPlane {
    gf_queue_plane spec;
    // gf_cuda_queue_create's plane: keep the pixel limits gf_get_frame_transform_at derives (FLT_MAX / 1 for float types, which
    // spec.max_value cannot express) instead of writing spec.max_value to them
    bool derived_limits;
    gf_stab_config stab;                  // the queue's, with the plane's pixel type and background (set by create_queue)
    int group;                            // index into gf_cuda_queue::groups (-1 until create_queue)
};

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
    std::vector<QPlane> planes;           // the layout: 1-4 planes
    std::vector<gf_buffer_desc> in_protos, out_protos;   // per plane
    std::vector<std::vector<size_t>> groups;   // plane indices of each group, in plane order
};

namespace {
int finish_slot(gf_cuda_queue* q, QSlot& s) {
    if (!s.busy) return GF_OK;
    CK(&q->last_error, cudaEventSynchronize(s.done.get()));
    s.busy = false;
    return GF_OK;
}

// A slot's stream, event, device table + verdict word, mesh staging and checksum word.
int init_slot(QSlot& s, size_t max_rows) {
    CK(nullptr, create_stream(s.stream));
    CK(nullptr, create_event(s.done));
    const cudaStream_t st = s.stream.get();
    CK(nullptr, s.d_mat.reserve(max_rows * GF_MATRIX_STRIDE, st));
    CK(nullptr, s.d_flags.reserve(1, st));
    CK(nullptr, s.h_mesh.reserve(GF_MESH_MAX_LEN, st));
    CK(nullptr, s.d_mesh.reserve(GF_MESH_MAX_LEN, st));
    CK(nullptr, s.d_sum.reserve(1, st));
    CK(nullptr, s.h_sum.reserve(1, st));
    *s.h_sum.ptr = 0;
    return GF_OK;
}

int enqueue_checksum_rows(const gf_checksum_plane* d, size_t n, uint64_t* out_dev, cudaStream_t st, std::string* err) {
    if (!d || !out_dev || n < 1 || n > 4) return fail(err, GF_ERR_BAD_PARAMS, "checksum: 1..4 descriptors and an output word");
    ChecksumRows P; memset(&P, 0, sizeof(P));
    P.n = (int)n;
    unsigned long long bytes = 0;
    for (size_t k = 0; k < n; ++k) {
        if (!d[k].ptr && d[k].rows && d[k].row_bytes) return fail(err, GF_ERR_BAD_PARAMS, "checksum: descriptor " + std::to_string(k) + " has no pointer");
        P.ptr[k] = static_cast<const uint8_t*>(d[k].ptr);
        P.row_bytes[k] = d[k].row_bytes; P.stride[k] = d[k].stride;
        P.first_row[k + 1] = P.first_row[k] + d[k].rows;
        P.first_byte[k] = bytes;
        bytes += (unsigned long long)d[k].rows * d[k].row_bytes;
    }
    P.end = bytes & ~3ull;
    CK(err, cudaMemsetAsync(out_dev, 0, sizeof(uint64_t), st));
    if (P.end) checksum_rows_kernel<<<132 * 4, 256, 0, st>>>(P, reinterpret_cast<unsigned long long*>(out_dev));
    CK(err, cudaGetLastError());
    return GF_OK;
}

int ceil_div(int a, int b) { return (a + b - 1) / b; }
bool same_shape(const gf_buffer_desc& a, const gf_buffer_desc& b) {
    return a.width == b.width && a.height == b.height && a.stride == b.stride && a.kind == b.kind;
}

using QueuePtr = std::unique_ptr<gf_cuda_queue, Deleter<gf_cuda_queue_destroy>>;

// Both creates, once the layout (planes, prototypes) is in `q`: the planes' stab configs and groups, gyro upload, the slots with one
// context per group (created for the group's first plane) and the HOST staging.
int create_queue(QueuePtr q, gf_cuda_queue** out) {
    const gf_queue_config& cfg = q->cfg;
    for (size_t i = 0; i < q->planes.size(); ++i) {
        QPlane& qp = q->planes[i];
        qp.stab = cfg.stab; qp.stab.pixel_type = qp.spec.pixel_type;
        memcpy(qp.stab.background, qp.spec.background, sizeof(qp.stab.background));
        for (size_t k = 0; k < q->groups.size() && qp.group < 0; ++k) {
            const gf_queue_plane& o = q->planes[q->groups[k][0]].spec;
            if (o.pixel_type == qp.spec.pixel_type && o.w_div == qp.spec.w_div && o.h_div == qp.spec.h_div) qp.group = (int)k;
        }
        if (qp.group < 0) { qp.group = (int)q->groups.size(); q->groups.emplace_back(); }
        q->groups[(size_t)qp.group].push_back(i);
    }
    CK(nullptr, cudaSetDevice(cfg.device));
    if (cfg.pin_numa) (void)gf_cuda_bind_thread_to_device(cfg.device);      // before any page-locked staging is allocated
    gf_cuda_gyro* gyro = nullptr;
    int rc = gf_cuda_gyro_upload(&gyro, cfg.device, &q->cp);
    if (rc != GF_OK) return rc;
    q->gyro.reset(gyro);
    q->max_rows = (size_t)(q->cp.width > q->cp.height ? q->cp.width : q->cp.height);
    q->slots.resize((size_t)cfg.depth);
    for (QSlot& s : q->slots) {
        if ((rc = init_slot(s, q->max_rows)) != GF_OK) return rc;
        for (const std::vector<size_t>& grp : q->groups) {
            const QPlane& qp = q->planes[grp[0]];
            gf_buffer_desc bi = q->in_protos[grp[0]], bo = q->out_protos[grp[0]];
            if (bi.kind == GF_BUF_HOST) bi.kind = GF_BUF_DEVICE;      // the context sees the slot's device copies of HOST planes
            if (bo.kind == GF_BUF_HOST) bo.kind = GF_BUF_DEVICE;
            gf_kernel_params kp; memset(&kp, 0, sizeof(kp));          // a template good enough for gf_cuda_create's validation
            kp.matrix_count = 1;
            rc = gf_get_frame_transform_at(&qp.stab, &q->cp, &bi, &bo, nullptr, 0, 0.0, 0, 1.0, &kp);
            if (rc != GF_OK) return fail(nullptr, rc, "plane " + std::to_string(grp[0]) + ": gf_get_frame_transform_at failed");
            gf_cuda_ctx* ctx = nullptr;
            rc = gf_cuda_create(&ctx, cfg.device, &kp, qp.spec.pixel_type, cfg.distortion_model, cfg.digital_lens, &bi, &bo, 0);
            if (rc != GF_OK) return rc;
            s.group_ctx.emplace_back(ctx);
        }
        CK(nullptr, s.staging.reserve(q->planes.size(), q->in_protos.data(), q->out_protos.data(), s.stream.get()));
    }
    *out = q.release();
    return GF_OK;
}

// Both submits, after their own argument checks: slot, producer, mesh, every plane's KernelParams, HOST staging, one planes call per
// group, checksum, download, event, FIFO.
int submit_frame(gf_cuda_queue* q, size_t frame, double timestamp_ms, size_t n_planes, const gf_buffer_desc* in, const gf_buffer_desc* out,
                 const float* mesh, size_t mesh_len, int fill_with_background) {
    std::string* const err = &q->last_error;
    if (n_planes != q->planes.size()) return fail(err, GF_ERR_BAD_PARAMS, "n_planes differs from the queue's layout (" + std::to_string(q->planes.size()) + ")");
    if (mesh_len > GF_MESH_MAX_LEN) return fail(err, GF_ERR_BUFFER_TOO_SMALL, "Buffer size mismatch buf_mesh_data");
    CK(err, cudaSetDevice(q->cfg.device));
    QSlot& s = q->slots[(size_t)q->next];
    if (s.busy) return fail(err, GF_ERR_BAD_PARAMS, "queue full: gf_cuda_queue_wait for the oldest frame first");
    int rc = s.staging.check(n_planes, in, out, err);
    if (rc != GF_OK) return rc;
    const cudaStream_t st = s.stream.get();
    nvtxRangePushA("gf_queue_submit");
    struct PopRange { ~PopRange() { nvtxRangePop(); } } pop_range;
    // one table + verdict for every plane: each plane's Stabilization is sized with the frame (rendering/mod.rs:514)
    gf_kernel_params kp0; size_t rows = 0; double fov = 1.0, minimal_fov = 1.0;
    rc = gf_cuda_frame_transform_dev_flagged(q->gyro.get(), &q->cp, timestamp_ms, frame, &kp0, s.d_mat.ptr, q->max_rows, s.d_flags.ptr,
                                             &rows, &fov, &minimal_fov, (void*)st);
    if (rc != GF_OK) return fail(err, rc, "gf_cuda_frame_transform_dev_flagged failed");
    q->launches++;
    const float* mesh_dev = nullptr;
    if (mesh && mesh_len) {
        memcpy(s.h_mesh.ptr, mesh, mesh_len * sizeof(float));
        CK(err, cudaMemcpyAsync(s.d_mesh.ptr, s.h_mesh.ptr, mesh_len * sizeof(float), cudaMemcpyHostToDevice, st));
        mesh_dev = s.d_mesh.ptr;
    }
    // the per-buffer half, per plane, as rendering/mod.rs:531-541 completes it before process_pixels
    gf_kernel_params kp[4];
    gf_buffer_desc din[4], dout[4];
    for (size_t i = 0; i < n_planes; ++i) {
        const QPlane& qp = q->planes[i];
        kp[i] = kp0;
        rc = gf_get_frame_transform_at(&qp.stab, &q->cp, &in[i], &out[i], mesh, mesh_len, timestamp_ms, frame, minimal_fov, &kp[i]);
        if (rc != GF_OK) return fail(err, rc, "plane " + std::to_string(i) + ": gf_get_frame_transform_at failed");
        if (!qp.derived_limits) kp[i].pixel_value_limit = kp[i].max_pixel_value = qp.spec.max_value;
        kp[i].plane_index = (int32_t)i;
        if (fill_with_background) kp[i].flags |= GF_FLAG_FILL_WITH_BACKGROUND;
    }
    // from here on, copies from the caller's HOST buffers may be queued: a failure waits for them before it returns
    struct WaitOnFailure { cudaStream_t st; bool ok; ~WaitOnFailure() { if (!ok) { (void)cudaStreamSynchronize(st); (void)cudaGetLastError(); } } } wait_on_failure{st, false};
    if ((rc = s.staging.upload(n_planes, in, out, kp, q->cfg.checksum != 0, st, err, din, dout)) != GF_OK) return rc;
    // each group through the planes path: its planner fuses the planes whose KernelParams agree, the rest get a warp each
    for (size_t g = 0; g < q->groups.size(); ++g) {
        const std::vector<size_t>& grp = q->groups[g];
        gf_buffer_desc gi[4], go[4]; gf_kernel_params gp[4];
        for (size_t j = 0; j < grp.size(); ++j) { gi[j] = din[grp[j]]; go[j] = dout[grp[j]]; gp[j] = kp[grp[j]]; }
        gf_cuda_ctx* const ctx = s.group_ctx[g].get();
        const unsigned long long l0 = gf_cuda_launch_count(ctx);
        rc = gf_cuda_undistort_planes_dev_flagged(ctx, grp.size(), gi, go, gp, s.d_mat.ptr, rows, mesh_dev, mesh_dev ? mesh_len : 0, s.d_flags.ptr, (void*)st);
        if (rc != GF_OK) return fail(err, rc, "plane " + std::to_string(grp[0]) + ": " + gf_cuda_last_error(ctx));
        q->launches += gf_cuda_launch_count(ctx) - l0;
    }
    if (q->cfg.checksum) {           // every plane's first min(len, height * stride) bytes: whole rows, then the rest of a short last row
        gf_checksum_plane d[8]; size_t nd = 0;
        for (size_t i = 0; i < n_planes; ++i) {
            const size_t stride = (size_t)dout[i].stride, nr = std::min((size_t)dout[i].height, dout[i].len / stride);
            const size_t tail = std::min(dout[i].len, (size_t)dout[i].height * stride) - nr * stride;
            d[nd++] = { dout[i].ptr, stride, stride, nr };
            if (tail) d[nd++] = { static_cast<const uint8_t*>(dout[i].ptr) + nr * stride, tail, tail, 1 };
        }
        if ((rc = enqueue_checksum_rows(d, nd, s.d_sum.ptr, st, err)) != GF_OK) return rc;
        q->launches++;
        CK(err, cudaMemcpyAsync(s.h_sum.ptr, s.d_sum.ptr, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    }
    if ((rc = s.staging.download(n_planes, out, kp, st, err)) != GF_OK) return rc;
    CK(err, cudaEventRecord(s.done.get(), st));
    wait_on_failure.ok = true;
    s.busy = true; s.frame = frame;
    q->fifo.push_back(q->next);
    q->next = (q->next + 1) % (int)q->slots.size();
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

// One whole-row descriptor of 64 KiB rows and one for the rest: the rows kernel gives each block whole rows.
GF_API int gf_cuda_checksum_dev(const void* ptr_dev, size_t len, uint64_t* out_dev, void* cu_stream) {
    if (!ptr_dev || !out_dev) return GF_ERR_BAD_PARAMS;
    const size_t row = (size_t)1 << 16, rows = len >> 16, tail = len & (row - 1);
    const gf_checksum_plane d[2] = { { ptr_dev, row, row, rows }, { static_cast<const uint8_t*>(ptr_dev) + rows * row, tail, tail, 1 } };
    return enqueue_checksum_rows(d, tail ? 2 : 1, out_dev, (cudaStream_t)cu_stream, nullptr);
}

GF_API int gf_cuda_queue_create(gf_cuda_queue** out, const gf_queue_config* cfg, const gf_compute_params* cp,
                                const gf_buffer_desc* in_proto, const gf_buffer_desc* out_proto) {
    if (!out || !cfg || !cp || !in_proto || !out_proto) return GF_ERR_BAD_PARAMS;
    *out = nullptr;
    if (cfg->depth < 1 || cfg->depth > 16) return GF_ERR_BAD_PARAMS;
    QueuePtr q(new gf_cuda_queue());
    q->cfg = *cfg; q->cp = *cp;
    gf_queue_plane spec{cfg->stab.pixel_type, 1, 1, 0.0f, {}};     // the config's pixel type and background, full size
    memcpy(spec.background, cfg->stab.background, sizeof(spec.background));
    q->planes.push_back(QPlane{spec, true, {}, -1});
    q->in_protos.push_back(*in_proto); q->out_protos.push_back(*out_proto);
    return create_queue(std::move(q), out);
}

GF_API int gf_cuda_queue_create_planes(gf_cuda_queue** out, const gf_queue_config* cfg, const gf_compute_params* cp, size_t n_planes,
                                       const gf_queue_plane* planes, const gf_buffer_desc* in_protos, const gf_buffer_desc* out_protos) {
    if (!out || !cfg || !cp || !planes || !in_protos || !out_protos) return fail(nullptr, GF_ERR_BAD_PARAMS, "null argument");
    *out = nullptr;
    if (n_planes < 1 || n_planes > 4) return fail(nullptr, GF_ERR_BAD_PARAMS, "n_planes must be 1..4");
    if (cfg->depth < 1 || cfg->depth > 16) return fail(nullptr, GF_ERR_BAD_PARAMS, "depth must be 1..16");
    QueuePtr q(new gf_cuda_queue());
    q->cfg = *cfg; q->cp = *cp;
    // everything checkable on the host first: nothing touches the device before the layout is known to be good
    for (size_t i = 0; i < n_planes; ++i) {
        const gf_queue_plane& pl = planes[i];
        const gf_buffer_desc& bi = in_protos[i], &bo = out_protos[i];
        const std::string name = "plane " + std::to_string(i) + ": ";
        if ((pl.w_div != 1 && pl.w_div != 2) || (pl.h_div != 1 && pl.h_div != 2)) return fail(nullptr, GF_ERR_BAD_PARAMS, name + "w_div and h_div must be 1 or 2");
        if (!gf_combo_supported(pl.pixel_type, cfg->distortion_model, cfg->digital_lens, cfg->stab.interpolation))
            return fail(nullptr, GF_ERR_BAD_PARAMS, name + "no kernel for this (pixel type, lens, digital lens, interpolation)");
        if ((bi.kind != GF_BUF_HOST && bi.kind != GF_BUF_DEVICE) || bi.kind != in_protos[0].kind || bo.kind != bi.kind || !bi.ptr || !bo.ptr)
            return fail(nullptr, GF_ERR_BAD_PARAMS, name + "buffers must all be HOST or all DEVICE, with a pointer");
        if ((pl.pixel_type == GF_PIX_UV8 || pl.pixel_type == GF_PIX_UV16) &&
            (bi.width != ceil_div(cfg->stab.width, pl.w_div) || bo.width != ceil_div(cfg->stab.output_width, pl.w_div)))
            return fail(nullptr, GF_ERR_BAD_PARAMS, name + "a UV plane is ceil(W / w_div) pixels wide");
        if (bo.stride < 1 || bo.height < 1 || bo.len < (size_t)bo.height * (size_t)bo.stride)
            return fail(nullptr, GF_ERR_BAD_PARAMS, name + "the output buffer holds fewer than height rows of stride bytes");
        q->planes.push_back(QPlane{pl, false, {}, -1});
    }
    q->in_protos.assign(in_protos, in_protos + n_planes); q->out_protos.assign(out_protos, out_protos + n_planes);
    return create_queue(std::move(q), out);
}

GF_API int gf_cuda_queue_submit(gf_cuda_queue* q, size_t frame, double timestamp_ms, const gf_buffer_desc* in, const gf_buffer_desc* out,
                                const float* mesh, size_t mesh_len) {
    if (!q || !in || !out) return fail(q ? &q->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    return submit_frame(q, frame, timestamp_ms, 1, in, out, mesh, mesh_len, 0);
}

GF_API int gf_cuda_queue_submit_planes(gf_cuda_queue* q, size_t frame, double timestamp_ms, size_t n_planes, const gf_buffer_desc* in,
                                       const gf_buffer_desc* out, const float* mesh, size_t mesh_len, int fill_with_background) {
    if (!q || !in || !out) return fail(q ? &q->last_error : nullptr, GF_ERR_BAD_PARAMS, "null argument");
    std::string* const err = &q->last_error;
    for (size_t i = 0; i < std::min(n_planes, q->planes.size()); ++i) {      // a count other than the layout's: submit_frame refuses it
        const std::string name = "plane " + std::to_string(i) + ": ";
        if (in[i].kind != in[0].kind || out[i].kind != in[0].kind) return fail(err, GF_ERR_BAD_PARAMS, name + "HOST and DEVICE buffers mixed in one frame");
        if (!same_shape(in[i], q->in_protos[i]) || !same_shape(out[i], q->out_protos[i]) || !in[i].ptr || !out[i].ptr)
            return fail(err, GF_ERR_BAD_PARAMS, name + "buffer size, stride or kind differs from the prototype's");
        if (out[i].len < (size_t)out[i].height * (size_t)out[i].stride)
            return fail(err, GF_ERR_BAD_PARAMS, name + "the output buffer holds fewer than height rows of stride bytes");
    }
    return submit_frame(q, frame, timestamp_ms, n_planes, in, out, mesh, mesh_len, fill_with_background);
}

GF_API int gf_cuda_checksum_planes_dev(const gf_checksum_plane* planes, size_t n, uint64_t* out_dev, void* cu_stream) {
    return enqueue_checksum_rows(planes, n, out_dev, (cudaStream_t)cu_stream, nullptr);
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
