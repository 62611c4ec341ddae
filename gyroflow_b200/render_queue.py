"""Frame-sharded render queue: the multi-GPU shape of the path (SURVEY.md §8e).

Frames are independent units (FrameTransform::at_timestamp depends only on immutable params + the timestamp,
src/core/stabilization/frame_transform.rs:165), so frame i goes to rank i % world and there is NO data-path collective.
The only communication is one broadcast, at job start, of the tables every rank needs (KernelParams template,
lens coefficients, per-frame matrix tables / quaternion tracks) from rank 0 — NCCL over NVLink on GPUs, gloo in the CPU
tests.  The reference has no counterpart: its render queue runs whole jobs in parallel (rendering/render_queue.rs:550-612)
but each job is a sequential decode -> warp -> encode loop on one device (rendering/mod.rs:451).
"""
import ctypes as C
from dataclasses import dataclass
from typing import Tuple

import numpy as np

from . import abi
from .backend import GyroflowCoreError, check_call


class RenderQueue:
    """One GPU's render queue (gf_cuda_queue, csrc/render_queue.cu): `depth` frames in flight, each
    producer kernel -> [H2D] -> warp -> [checksum] -> [D2H] on its own stream; results come back in submission order.

    bench.py and the multi-GPU tests drive this class: rank r of a world of G submits frames r, r + G, r + 2G, ...
    (shard_frames) and the per-frame checksums are gathered in frame order (gather_results)."""

    def __init__(self, compute_params, stab: abi.StabConfig, distortion_model: str, digital_lens, in_proto, out_proto,
                 device=0, depth=4, pin_numa=True, checksum=False, planes=None):
        self._lib = abi.load_library()
        self.cp = compute_params                      # keeps the arrays alive
        cfg = abi.QueueConfig()
        cfg.device = device
        cfg.distortion_model = abi.LENS[distortion_model]
        cfg.digital_lens = abi.LENS[digital_lens] if digital_lens else 0
        cfg.depth, cfg.pin_numa, cfg.checksum = depth, int(pin_numa), int(checksum)
        cfg.stab = stab
        self.depth = depth
        self.in_flight = 0
        self.n_planes = 0 if planes is None else len(planes)
        h = C.c_void_p()
        if planes is None:
            i, o = in_proto.to_c(), out_proto.to_c()
            rc = self._lib.gf_cuda_queue_create(C.byref(h), C.byref(cfg), C.byref(compute_params.c), C.byref(i), C.byref(o))
            what = "gf_cuda_queue_create"
        else:
            n = len(planes)
            specs = (abi.QueuePlane * n)(*planes)
            ins = (abi.BufferDesc * n)(*[b.to_c() for b in in_proto])
            outs = (abi.BufferDesc * n)(*[b.to_c() for b in out_proto])
            rc = self._lib.gf_cuda_queue_create_planes(C.byref(h), C.byref(cfg), C.byref(compute_params.c), n, specs, ins, outs)
            what = "gf_cuda_queue_create_planes"
        check_call(rc, what)
        self._h = h

    @classmethod
    def for_planes(cls, compute_params, stab: abi.StabConfig, distortion_model: str, digital_lens, planes, in_protos, out_protos, **kw):
        """A queue for decoder frames of 1-4 planes (gf_cuda_queue_create_planes): `planes` are abi.QueuePlane (PlaneLayout.to_c of
        layout()), `in_protos` / `out_protos` one BufferDescription per plane.  submit() then takes a list of Buffers per frame."""
        return cls(compute_params, stab, distortion_model, digital_lens, in_protos, out_protos, planes=planes, **kw)

    def _err(self, rc, what):
        return GyroflowCoreError(rc, what + ": " + (self._lib.gf_cuda_queue_last_error(self._h) or b"").decode())

    def submit(self, frame: int, timestamp_ms: float, buffers, mesh=None, fill_with_background=False):
        """Enqueue one frame (a planes queue: a list of Buffers, one per plane).  The queue must have a free slot (in_flight < depth):
        call wait() first otherwise.  fill_with_background: the render loop's per-frame flag, planes queues only (a one-plane queue
        takes FILL_WITH_BACKGROUND through StabConfig.base_flags)."""
        m = None if mesh is None else np.ascontiguousarray(mesh, dtype=np.float32)
        mp, mn = (m.ctypes.data if m is not None and m.size else None), (m.size if m is not None else 0)
        if self.n_planes:
            n = len(buffers)
            ins = (abi.BufferDesc * n)(*[b.input.to_c() for b in buffers])
            outs = (abi.BufferDesc * n)(*[b.output.to_c() for b in buffers])
            rc = self._lib.gf_cuda_queue_submit_planes(self._h, frame, timestamp_ms, n, ins, outs, mp, mn, int(fill_with_background))
            what = "gf_cuda_queue_submit_planes"
        else:
            if fill_with_background:
                raise ValueError("a one-plane queue takes FILL_WITH_BACKGROUND through StabConfig.base_flags")
            i, o = buffers.input.to_c(), buffers.output.to_c()
            rc = self._lib.gf_cuda_queue_submit(self._h, frame, timestamp_ms, C.byref(i), C.byref(o), mp, mn)
            what = "gf_cuda_queue_submit"
        if rc != 0:
            raise self._err(rc, what)
        self.in_flight += 1

    def wait(self):
        """Block until the oldest in-flight frame is finished; returns (frame, checksum)."""
        f = C.c_size_t(); s = C.c_uint64()
        rc = self._lib.gf_cuda_queue_wait(self._h, C.byref(f), C.byref(s))
        if rc != 0:
            raise self._err(rc, "gf_cuda_queue_wait")
        self.in_flight -= 1
        return int(f.value), int(s.value)

    def render(self, frames, timestamp_of, buffers_of, mesh_of=None, fill_with_background=False):
        """Run `frames` (an iterable of frame indices) through the queue keeping it full; returns {frame: checksum} in frame order.
        buffers_of(f): the frame's Buffers, or for a planes queue its list of per-plane Buffers."""
        out = {}
        for f in frames:
            if self.in_flight == self.depth:
                k, v = self.wait(); out[k] = v
            self.submit(f, timestamp_of(f), buffers_of(f), mesh_of(f) if mesh_of else None, fill_with_background)
        while self.in_flight:
            k, v = self.wait(); out[k] = v
        return dict(sorted(out.items()))

    def drain(self):
        rc = self._lib.gf_cuda_queue_drain(self._h)
        if rc != 0:
            raise self._err(rc, "gf_cuda_queue_drain")
        self.in_flight = 0

    @property
    def launch_count(self):
        return int(self._lib.gf_cuda_queue_launches(self._h))

    def close(self):
        if getattr(self, "_h", None):
            self._lib.gf_cuda_queue_destroy(self._h); self._h = None

    def __del__(self):
        try: self.close()
        except Exception: pass


def checksum_host(buf: np.ndarray) -> int:
    """The queue's per-frame checksum on the host: sum(word[i] * (2 i + 1)) mod 2^64 over the buffer's 32-bit words."""
    w = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
    w = w[: w.size // 4 * 4].view(np.uint32).astype(np.uint64)
    k = np.arange(w.size, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    with np.errstate(over="ignore"):
        return int((w * k).sum(dtype=np.uint64))


def plane_rows(buf: np.ndarray, row_bytes: int, stride: int, rows: int) -> np.ndarray:
    """The bytes a gf_checksum_plane descriptor names: `rows` rows of `row_bytes` bytes, `stride` bytes apart, concatenated."""
    b = np.ascontiguousarray(buf).view(np.uint8).reshape(-1)
    if rows == 0 or row_bytes == 0:
        return np.zeros(0, np.uint8)
    idx = np.arange(rows, dtype=np.int64)[:, None] * stride + np.arange(row_bytes, dtype=np.int64)[None, :]
    return b[idx.reshape(-1)]


def checksum_planes_host(descs) -> int:
    """The multi-plane checksum (gf_cuda_checksum_planes_dev, a planes queue's frame checksum) on the host: descs = [(buffer,
    row_bytes, stride, rows)]; checksum_host of their rows concatenated in order.  One (buf, stride, stride, rows) descriptor is
    checksum_host of the buffer's first rows * stride bytes."""
    parts = [plane_rows(b, rb, st, r) for b, rb, st, r in descs]
    return checksum_host(np.concatenate(parts) if parts else np.zeros(0, np.uint8))


# ---- decoder formats -> plane layouts: create_planes_proc! in the reference's rendering/mod.rs:563-651 -------------------------------
@dataclass(frozen=True)
class PlaneLayout:
    """One plane of a decoder format: its pixel type, size fraction of the frame (ceil(W / w_div) x ceil(H / h_div)), the value the
    render loop writes to pixel_value_limit / max_pixel_value, and the component list (`$yuvi`) from_rgb_color converts the background
    with — that conversion stays with the caller."""
    pixel_type: str
    w_div: int
    h_div: int
    max_value: float
    components: Tuple[int, ...]

    def size(self, width, height):
        return (-(-width // self.w_div), -(-height // self.h_div))

    def to_c(self, background=(0.0, 0.0, 0.0, 0.0)) -> abi.QueuePlane:
        p = abi.QueuePlane()
        p.pixel_type, p.w_div, p.h_div, p.max_value = abi.PIXEL_TYPES[self.pixel_type][0], self.w_div, self.h_div, self.max_value
        p.background[:] = [float(v) for v in background]
        return p


def _yuv(luma, chroma, w_div, h_div, max_value, uv_components=None, alpha=False):
    if chroma.startswith("UV"):
        return (PlaneLayout(luma, 1, 1, max_value, (0,)), PlaneLayout(chroma, w_div, h_div, max_value, uv_components))
    planes = [PlaneLayout(luma, 1, 1, max_value, (0,))] + [PlaneLayout(chroma, w_div, h_div, max_value, (c,)) for c in (1, 2)]
    return tuple(planes + ([PlaneLayout(luma, 1, 1, max_value, (3,))] if alpha else []))


DECODER_FORMATS = {
    "nv12": _yuv("Luma8", "UV8", 2, 2, 255.0, (1, 2)),
    "nv21": _yuv("Luma8", "UV8", 2, 2, 255.0, (2, 1)),
    "yuv420p": _yuv("Luma8", "Luma8", 2, 2, 255.0),
    "yuvj420p": _yuv("Luma8", "Luma8", 2, 2, 255.0),
    # the reference keeps 65535 for the 10-bit P0xx formats too (their samples sit in the high bits)
    **{"p%s%s" % (s, b): _yuv("Luma16", "UV16", wd, hd, 65535.0, (1, 2))
       for s, (wd, hd) in (("0", (2, 2)), ("2", (2, 1)), ("4", (1, 1))) for b in ("10", "16")},
    **{"yuv4%sp%s" % (s, b): _yuv("Luma16", "Luma16", wd, hd, float((1 << int(b)) - 1))
       for s, (wd, hd) in (("20", (2, 2)), ("22", (2, 1)), ("44", (1, 1))) for b in ("10", "12", "14", "16")},
    **{"yuva444p%s" % b: _yuv("Luma16", "Luma16", 1, 1, float((1 << int(b)) - 1), alpha=True) for b in ("10", "12", "16")},
    # planes G, B, R(, A) in ffmpeg's order; from_rgb_color takes background components 2, 0, 1(, 3) for them
    "gbrapf32": tuple(PlaneLayout("R32f", 1, 1, 255.0, (c,)) for c in (2, 0, 1, 3)),
    "gbrpf32": tuple(PlaneLayout("R32f", 1, 1, 255.0, (c,)) for c in (2, 0, 1)),
}


def layout(fmt: str, width: int, height: int):
    """The planes of a decoder frame of format `fmt` (ffmpeg's name, case-insensitive, "le" suffix optional) and size width x height:
    a list of (PlaneLayout, (plane width, plane height)) in plane order."""
    key = fmt.lower()
    if key not in DECODER_FORMATS and key.endswith("le"):
        key = key[:-2]
    if key not in DECODER_FORMATS:
        raise KeyError("no plane layout for decoder format %r" % fmt)
    return [(pl, pl.size(width, height)) for pl in DECODER_FORMATS[key]]


def shard_frames(n_frames, world, rank):
    """Frame indices owned by `rank`: round-robin, so every rank sees the same mix of timestamps."""
    return list(range(rank, n_frames, world))


def frame_owner(frame, world):
    return frame % world


def params_to_tensor(p, torch):
    """KernelParams (368 B) as a uint8 tensor (for the broadcast)."""
    raw = C.string_at(C.byref(p), C.sizeof(abi.KernelParams))
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).clone()


def params_from_tensor(t):
    p = abi.KernelParams()
    raw = bytes(t.cpu().numpy().tobytes())
    C.memmove(C.byref(p), raw, C.sizeof(abi.KernelParams))
    return p


def broadcast_tables(params, matrices, dist, torch, device, src=0):
    """One-time broadcast of the job's tables from `src`.  `params`/`matrices` are only read on the source rank;
    every rank passes the expected matrices shape.  Returns (KernelParams, matrices tensor on `device`)."""
    rank = dist.get_rank()
    pt = params_to_tensor(params, torch).to(device) if rank == src else torch.empty(C.sizeof(abi.KernelParams), dtype=torch.uint8, device=device)
    shape = torch.tensor(list(matrices.shape) if rank == src else [0, 0, 0], dtype=torch.int64, device=device)
    dist.broadcast(shape, src=src)
    mt = (torch.as_tensor(np.ascontiguousarray(matrices, dtype=np.float32)).to(device) if rank == src
          else torch.empty(tuple(int(v) for v in shape.tolist()), dtype=torch.float32, device=device))
    dist.broadcast(pt, src=src)
    dist.broadcast(mt, src=src)
    return params_from_tensor(pt), mt


def _as_i64(v):
    v &= (1 << 64) - 1
    return v - (1 << 64) if v >= (1 << 63) else v


def gather_results(local, dist, torch, device, dst=0):
    """Collect {frame: value} dicts (small per-frame results such as 64-bit checksums) on every rank, restoring frame order."""
    local = {k: _as_i64(int(v)) for k, v in local.items()}
    world = dist.get_world_size()
    keys = torch.tensor(sorted(local), dtype=torch.int64, device=device)
    vals = torch.tensor([local[k] for k in sorted(local)], dtype=torch.int64, device=device)
    n = torch.tensor([keys.numel()], dtype=torch.int64, device=device)
    ns = [torch.zeros(1, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(ns, n)
    m = int(max(int(v.item()) for v in ns))
    pad = lambda t: torch.cat([t, torch.full((m - t.numel(),), -1, dtype=torch.int64, device=device)])
    ks = [torch.empty(m, dtype=torch.int64, device=device) for _ in range(world)]
    vs = [torch.empty(m, dtype=torch.int64, device=device) for _ in range(world)]
    dist.all_gather(ks, pad(keys)); dist.all_gather(vs, pad(vals))
    out = {}
    for k, v in zip(ks, vs):
        for a, b in zip(k.tolist(), v.tolist()):
            if a >= 0: out[a] = b & ((1 << 64) - 1)
    return dict(sorted(out.items()))
