"""The frame-sharded render queue (gf_cuda_queue_*, csrc/render_queue.cu; SURVEY §8e): per frame, on the device and without a host
sync, FrameTransform::at_timestamp (producer kernel + trust verdict) -> warp; `depth` frames in flight; results in submission order.

Parity: every frame's bytes (and the queue's device-side checksum) against the oracle run on the table the device producer wrote
for that timestamp (read back through gf_cuda_frame_transform_dev, the same deterministic kernel).  That table is itself checked
against the host producer (gf_frame_transform_at_timestamp: IBIS / OIS columns bit-identical, the rest within 1 f32 ulp), and
tests/test_device_producer.py checks the host producer against the numpy restatement, so a wrong device table cannot pass as its
own reference.  The 2-rank test renders frames `rank::2` of one job on two processes and gathers the per-frame checksums in frame order — over NCCL when the box has two GPUs,
over gloo with both ranks on GPU 0 otherwise (the data path has no collective either way)."""
import ctypes as C
import os
import socket

import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import abi, render_queue, synth
from tests import cases, oracle_lib, producer_cases

pytestmark = pytest.mark.gpu

W, H = 640, 360
FPS = 60.0


def _job(pix="RGBA8", lens="opencv_fisheye", digital=None, w=W, h=H, out_stride=None, **cpkw):
    p = synth.base_kernel_params(w, h, pixel_type=pix, lens=lens, digital_lens=digital, out_stride=out_stride)
    org, sm = cases.gyro()
    cp = g.ComputeParams(p, org, sm, **cpkw)
    return p, cp, g.stab_config(p, pix, digital_lens=digital)


def _expected(p, cp, st, dg, mats_dev, ts, frame, src, pix, lens, digital, bufs, mesh=None, fill=0):
    """The frame as the reference would render it from the table the device producer writes for (ts, frame), into an output buffer
    whose bytes are all `fill` before."""
    kp, rows = dg.frame_transform(ts, mats_dev.data_ptr(), max(p.width, p.height), frame=frame)     # stream = 0: synchronous
    table = mats_dev.cpu().numpy()[:rows].copy()
    kp_h, table_h, _, _ = cp.at_timestamp(ts, frame)              # the host producer: same KernelParams, the same table to the bars
    assert bytes(kp) == bytes(kp_h)                               # of tests/test_device_producer.py
    producer_cases.compare_tables(table, table_h)
    g.get_frame_transform_at(st, cp, bufs, kp, mesh=mesh, frame=frame)
    want = np.full((p.output_height, p.output_stride), fill, np.uint8)
    assert oracle_lib.undistort_image(src, want, kp, pix, lens, digital, table, mesh) == 0
    return want


def test_queue_device_buffers_every_frame_matches_oracle():
    import torch
    pix, lens = "RGBA8", "opencv_fisheye"
    p, cp, st = _job()
    src = synth.synthetic_frame(W, H, pix, stride=p.stride)
    tsrc = torch.from_numpy(src).cuda()
    n = 12
    outs = [torch.zeros((H, p.output_stride), dtype=torch.uint8, device="cuda") for _ in range(n)]
    bufs = [g.Buffers(g.BufferDescription((W, H, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                      g.BufferDescription((W, H, p.output_stride), o.data_ptr(), length=o.numel())) for o in outs]
    q = g.RenderQueue(cp, st, lens, None, bufs[0].input, bufs[0].output, depth=4, checksum=True)
    ts_of = lambda f: 300.0 + f * (1000.0 / FPS)
    sums = q.render(range(n), ts_of, lambda f: bufs[f])
    assert list(sums) == list(range(n))                       # frame order restored
    assert q.launch_count == 4 * n                            # producer + warp (main + tail of the filtered pre-pass) + checksum per frame, nothing else
    q.close()
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(W, H), 14), dtype=torch.float32, device="cuda")
    seen = set()
    for f in range(n):
        want = _expected(p, cp, st, dg, mats, ts_of(f), f, src, pix, lens, None, bufs[f])
        got = outs[f].cpu().numpy()
        assert np.array_equal(got, want), "frame %d" % f
        assert sums[f] == render_queue.checksum_host(want)
        seen.add(sums[f])
    assert len(seen) == n                                     # distinct timestamps -> distinct frames
    dg.close()


@pytest.mark.parametrize("pix,lens,digital,extra", [
    ("RGBA8", "opencv_fisheye", None, {}),
    ("Luma16", "opencv_fisheye", "gopro_superview", {}),
    ("RGBAf", "sony", None, dict(stab=True, mesh=True)),          # IBIS rows from the spline producer + per-frame mesh: guarded / general kernel
    ("RGBA8", "opencv_fisheye", None, dict(stab="alternate")),     # packed kernel, consecutive slots alternate between verdicts 2 and 0
    # five fisheye lenses in turn: each slot's context sees all five (one radial-table eviction) and then its first lens again (a rebuild)
    ("RGBA8", "opencv_fisheye", None, dict(lenses=5, n=18)),
])
def test_queue_host_buffers_pipelined(pix, lens, digital, extra):
    import torch
    from tests.test_frame_transform import _stab
    n = extra.get("n", 9)
    kw = {}
    if extra.get("lenses"):
        p0 = synth.base_kernel_params(W, H)
        K = [p0.f[0], 0.0, p0.c[0], 0.0, p0.f[1], p0.c[1], 0.0, 0.0, 1.0]
        L = [dict(camera_matrix=K, distortion_coeffs=[0.05 - 0.03 * i, 0.01 * (i % 2), -0.002, 0.0005 * i] + [0.0] * 8) for i in range(extra["lenses"])]
        kw = dict(lens_per_frame=[L[f % len(L)] for f in range(n)])
    if extra.get("stab") == "alternate":      # spline points on even frames (counts differ), none on odd ones, frames 7 and 8 past the end
        stab = producer_cases.spline_stab([12, 0, 31, 0, 6, 0, 19], seed=8)
        kw = dict(camera_stab=stab, sync_offsets={500_000: 3.0, 800_000: -1.5, 1_200_000: 2.5})
    elif extra.get("stab"):
        kw = dict(camera_stab=_stab(n, H), per_frame_time_offsets=[0.25 * i for i in range(n)], sync_offsets={0: 1.0, 2_000_000: -2.0, 4_000_000: 0.5})
    p, cp, st = _job(pix, lens, digital, **kw)
    mesh = synth.synthetic_mesh(W, H) if extra.get("mesh") else None
    srcs = [torch.from_numpy(synth.synthetic_frame(W, H, pix, frame=i, stride=p.stride)).pin_memory() for i in range(3)]
    outs = [torch.zeros((H, p.output_stride), dtype=torch.uint8).pin_memory() for _ in range(n)]
    bufs = [g.Buffers(g.BufferDescription((W, H, p.stride), srcs[f % 3].numpy()), g.BufferDescription((W, H, p.output_stride), outs[f].numpy())) for f in range(n)]
    q = g.RenderQueue(cp, st, lens, digital, bufs[0].input, bufs[0].output, depth=3, checksum=True)
    ts_of = lambda f: 700.0 + f * (1000.0 / FPS)
    sums = q.render(range(n), ts_of, lambda f: bufs[f], (lambda f: mesh) if mesh is not None else None)
    q.close()
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(W, H), 14), dtype=torch.float32, device="cuda")
    for f in range(n):
        want = _expected(p, cp, st, dg, mats, ts_of(f), f, srcs[f % 3].numpy(), pix, lens, digital, bufs[f], mesh)
        assert np.array_equal(outs[f].numpy(), want), "frame %d" % f
        assert sums[f] == render_queue.checksum_host(want)
    if extra.get("stab") is True:
        assert np.abs(mats.cpu().numpy()[:H, 9:]).max() > 1.0       # the IBIS columns really were exercised
    if extra.get("stab") == "alternate":      # the verdict each slot's producer gave: IBIS rows on even frames up to 6, nothing else
        for f in range(n):
            _, table, _, _ = cp.at_timestamp(ts_of(f), f)
            assert producer_cases.table_flags_host(table) == (2 if f % 2 == 0 and f < 7 else 0), f
    dg.close()


@pytest.mark.parametrize("rect", [None, (24, 10, W - 40, H - 30)])
def test_queue_host_output_rows_with_padding(rect):
    """HOST output rows with 64 bytes of padding, every byte pre-filled with 0xA5: the bytes equal the oracle's render into the same
    pre-fill, the padding keeps its 0xA5, and the checksum the queue returns is that of the host buffer it hands back.  Without a rect the
    warp covers the buffer, so only the pixel rows come back; with one it does not, so the buffer is uploaded before the warp."""
    import torch
    pix, lens, n = "RGBA8", "opencv_fisheye", 6
    p, cp, st = _job(out_stride=W * 4 + 64)
    src = torch.from_numpy(synth.synthetic_frame(W, H, pix, stride=p.stride)).pin_memory()
    outs = [torch.full((H, p.output_stride), 0xA5, dtype=torch.uint8).pin_memory() for _ in range(n)]
    bufs = [g.Buffers(g.BufferDescription((W, H, p.stride), src.numpy()), g.BufferDescription((W, H, p.output_stride), o.numpy(), rect=rect))
            for o in outs]
    q = g.RenderQueue(cp, st, lens, None, bufs[0].input, bufs[0].output, depth=3, checksum=True)
    ts_of = lambda f: 500.0 + f * (1000.0 / FPS)
    sums = q.render(range(n), ts_of, lambda f: bufs[f])
    q.close()
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(W, H), 14), dtype=torch.float32, device="cuda")
    for f in range(n):
        got = outs[f].numpy()
        want = _expected(p, cp, st, dg, mats, ts_of(f), f, src.numpy(), pix, lens, None, bufs[f], fill=0xA5)
        assert np.array_equal(got, want), "frame %d" % f
        assert (got[:, W * 4:] == 0xA5).all(), "frame %d" % f
        assert sums[f] == render_queue.checksum_host(got), "frame %d" % f
    dg.close()


def test_thousand_frame_job_cfg5_shape():
    """BASELINE config 5's shape at a reduced frame size: 1000 frames with distinct timestamps through one queue, 6 in flight, results in
    frame order; every 40th frame against the oracle (bytes through the checksum), and no two neighbouring frames alike."""
    import torch
    p, cp, st = _job(w=480, h=270)
    w, h = 480, 270
    org, sm = synth.synthetic_gyro(1000 / FPS + 2.0)
    cp = g.ComputeParams(p, org, sm)
    src = synth.synthetic_frame(w, h, "RGBA8", stride=p.stride)
    tsrc = torch.from_numpy(src).cuda()
    ring = [torch.zeros((h, p.output_stride), dtype=torch.uint8, device="cuda") for _ in range(6)]
    mk = lambda f: g.Buffers(g.BufferDescription((w, h, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                             g.BufferDescription((w, h, p.output_stride), ring[f % 6].data_ptr(), length=ring[f % 6].numel()))
    q = g.RenderQueue(cp, st, "opencv_fisheye", None, mk(0).input, mk(0).output, depth=6, checksum=True)
    ts_of = lambda f: 200.0 + f * (1000.0 / FPS)
    sums = q.render(range(1000), ts_of, mk)
    q.close()
    assert list(sums) == list(range(1000))
    assert all(sums[f] != sums[f + 1] for f in range(999))
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(w, h), 14), dtype=torch.float32, device="cuda")
    for f in range(0, 1000, 40):
        want = _expected(p, cp, st, dg, mats, ts_of(f), f, src, "RGBA8", "opencv_fisheye", None, mk(f))
        assert sums[f] == render_queue.checksum_host(want), "frame %d" % f
    dg.close()


def test_queue_full_and_errors():
    import torch
    p, cp, st = _job()
    src = torch.zeros((H, p.stride), dtype=torch.uint8, device="cuda"); dst = torch.zeros((H, p.output_stride), dtype=torch.uint8, device="cuda")
    b = g.Buffers(g.BufferDescription((W, H, p.stride), src.data_ptr(), length=src.numel()), g.BufferDescription((W, H, p.output_stride), dst.data_ptr(), length=dst.numel()))
    q = g.RenderQueue(cp, st, "opencv_fisheye", None, b.input, b.output, depth=2)
    for bad in (g.BufferDescription((W, H, p.stride), None), g.BufferDescription((W, H, p.stride), 0, length=src.numel())):
        rc = q._lib.gf_cuda_queue_submit(q._h, 0, 100.0, C.byref(bad.to_c()), C.byref(b.output.to_c()), None, 0)
        assert rc == -1                                        # no buffer / a null pointer: GF_ERR_BAD_PARAMS, not a failed copy
    q.submit(0, 100.0, b); q.submit(1, 120.0, b)
    with pytest.raises(g.GyroflowCoreError):
        q.submit(2, 140.0, b)                                  # queue full: wait() first
    q.in_flight = 2
    assert q.wait()[0] == 0 and q.wait()[0] == 1
    with pytest.raises(g.GyroflowCoreError) as e:
        q.wait()
    assert e.value.kind == "NoStabilizationData"
    q.in_flight = 0
    q.close()


# ---- two ranks: frames rank::2 on each, checksums gathered in frame order ---------------------------------------------------------
N_FRAMES = 10


def _rank_worker(rank, world, port, n_gpus, outq):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev_index = rank % n_gpus
    torch.cuda.set_device(dev_index)
    if n_gpus >= world:
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev_index))
        cdev = torch.device("cuda", dev_index)
    else:                                                      # one GPU: both ranks share it, the bookkeeping collective runs on gloo
        dist.init_process_group("gloo", rank=rank, world_size=world)
        cdev = torch.device("cpu")
    # rank 0 owns the job description; one broadcast of the quaternion tracks (the only data every rank needs), SURVEY §8e
    p = synth.base_kernel_params(W, H)
    if rank == 0:
        org, sm = cases.gyro()
        ots, oq, sts, sq = (torch.from_numpy(np.ascontiguousarray(a)) for a in (org.ts, org.q, sm.ts, sm.q))
    else:
        n = len(cases.gyro()[0].ts)                           # shapes are part of the job description
        ots, oq, sts, sq = torch.zeros(n, dtype=torch.int64), torch.zeros((n, 4), dtype=torch.float64), torch.zeros(n, dtype=torch.int64), torch.zeros((n, 4), dtype=torch.float64)
    tensors = [t.to(cdev) for t in (ots, oq, sts, sq)]
    for t in tensors: dist.broadcast(t, src=0)
    ots, oq, sts, sq = (t.cpu().numpy() for t in tensors)
    cp = g.ComputeParams(p, synth.GyroTrack(ots, oq), synth.GyroTrack(sts, sq))
    st = g.stab_config(p, "RGBA8")
    src = synth.synthetic_frame(W, H, "RGBA8", stride=p.stride)
    tsrc = torch.from_numpy(src).cuda()
    mine = render_queue.shard_frames(N_FRAMES, world, rank)
    outs = {f: torch.zeros((H, p.output_stride), dtype=torch.uint8, device="cuda") for f in mine}
    mk = lambda f: g.Buffers(g.BufferDescription((W, H, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                             g.BufferDescription((W, H, p.output_stride), outs[f].data_ptr(), length=outs[f].numel()))
    q = g.RenderQueue(cp, st, "opencv_fisheye", None, mk(mine[0]).input, mk(mine[0]).output, device=dev_index, depth=3, checksum=True)
    local = q.render(mine, lambda f: 250.0 + f * (1000.0 / FPS), mk)
    q.close()
    allr = render_queue.gather_results(local, dist, torch, cdev)
    if rank == 0:
        outq.put((allr, dist.get_backend()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_ranks_render_a_sharded_job_and_match_the_oracle():
    import torch
    import torch.multiprocessing as mp
    n_gpus = torch.cuda.device_count()
    assert n_gpus >= 1
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    outq = ctx.Queue()
    procs = [ctx.Process(target=_rank_worker, args=(r, 2, port, n_gpus, outq)) for r in range(2)]
    for pr in procs: pr.start()
    got, backend = outq.get(timeout=300)
    for pr in procs:
        pr.join(timeout=120)
        assert pr.exitcode == 0
    assert backend == ("nccl" if n_gpus >= 2 else "gloo")
    assert list(got) == list(range(N_FRAMES))
    # every frame against the oracle, on this process's GPU
    p, cp, st = _job()
    src = synth.synthetic_frame(W, H, "RGBA8", stride=p.stride)
    dg = g.DeviceGyro(cp)
    mats = torch.zeros((max(W, H), 14), dtype=torch.float32, device="cuda")
    dst = np.zeros((H, p.output_stride), np.uint8)
    b = g.Buffers(g.BufferDescription((W, H, p.stride), src), g.BufferDescription((W, H, p.output_stride), dst))
    for f in range(N_FRAMES):
        want = _expected(p, cp, st, dg, mats, 250.0 + f * (1000.0 / FPS), f, src, "RGBA8", "opencv_fisheye", None, b)
        assert got[f] == render_queue.checksum_host(want), "frame %d rendered by rank %d" % (f, f % 2)
    dg.close()
