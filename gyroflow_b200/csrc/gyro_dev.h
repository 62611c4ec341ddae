// gyro_dev.h — the device-resident per-clip data behind gf_cuda_gyro (shared by frame_transform.cu and zoom_kernel.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstddef>
#include <vector>
#include "frame_geometry.cuh"
#include "c_abi_internal.h"

struct gf_cuda_gyro {
    int device = 0;
    gf::GrowBuf<int64_t> d_org_ts; gf::GrowBuf<double> d_org_q; size_t n_org = 0;       // quaternions (org track)
    gf::GrowBuf<int64_t> d_off_ts; gf::GrowBuf<double> d_off_ms; size_t n_offsets = 0;  // offsets_adjusted (multi-point sync), may be empty
    gf::GrowBuf<double> d_stab;                                                         // IBIS / OIS spline points of every frame, flat
    struct StabIndex { size_t ibis_pos, ibis_val, n_ibis, ois_pos, ois_val, n_ois; };
    std::vector<StabIndex> stab_index;                                                  // offsets into d_stab per frame
    gf::GrowBuf<double> d_mesh;                                                         // distorting meshes of every frame (point path), flat
    struct MeshIndex { size_t off, len; double header[9]; };                       // header: host copy of the mesh's first 9 values
    std::vector<MeshIndex> mesh_index;
    // verdict accumulator + ticket of frame_rows_kernel: a pool of pairs handed out round-robin, so that producer launches that overlap
    // on different streams (the render queue's slots) never share one
    static constexpr unsigned kScratchPairs = 64;
    gf::GrowBuf<unsigned> d_scratch; unsigned next_scratch = 0;
    gf::Stream stream;
    // ST-map jobs (gf_cuda_generate_stmaps_dev, and gf_cuda_generate_stmap as a job of one frame): the coordinate-mode warp context they
    // share, kept from job to job, and the end of the last job on its stream
    std::unique_ptr<gf_cuda_ctx, gf::Deleter<gf_cuda_destroy>> stmap_ctx;
    gf::Event stmap_done;
    // the last visual-features sync call (gf_cuda_sync_last_timing)
    double sync_host_ms = 0.0, sync_device_ms = 0.0; size_t sync_chunks = 0;

    // the stream of a call: the caller's `cu_stream`, or this object's own when it is NULL
    cudaStream_t stream_of(void* cu_stream) const { return cu_stream ? (cudaStream_t)cu_stream : stream.get(); }
    gf::Track org_track() const { return gf::Track{ d_org_ts.ptr, d_org_q.ptr, n_org }; }
    // the uploaded multi-point sync offsets; `scalar_ms` (gyro_offset_ms) applies when there are none
    gf::SyncOffsets sync_offsets(double scalar_ms) const { return gf::SyncOffsets{ d_off_ts.ptr, d_off_ms.ptr, n_offsets, scalar_ms }; }
    // this frame's IBIS / OIS spline points; false when the upload had no camera_stab entry for it
    bool frame_splines(size_t frame, gf::StabSplines& s) const {
        if (frame >= stab_index.size()) return false;
        const StabIndex& ix = stab_index[frame];
        s.ibis = gf::Spline3{ d_stab.ptr + ix.ibis_pos, d_stab.ptr + ix.ibis_val, ix.n_ibis };
        s.ois  = gf::Spline3{ d_stab.ptr + ix.ois_pos,  d_stab.ptr + ix.ois_val,  ix.n_ois };
        return true;
    }
    // this frame's distorting mesh (mesh_correction[frame].0) and its length, or nullptr when it has none of more than 9 values
    const double* frame_mesh(size_t frame, uint32_t& len) const {
        len = 0;
        if (!d_mesh.ptr || frame >= mesh_index.size() || mesh_index[frame].len <= 9) return nullptr;
        len = (uint32_t)mesh_index[frame].len;
        return d_mesh.ptr + mesh_index[frame].off;
    }
};
