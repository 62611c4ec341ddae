"""The per-frame table producer over every case of tests/producer_cases.py:

- the host producer (gf_frame_transform_at_timestamp) against the numpy restatement (CPU);
- the device producer (gf_cuda_frame_transform_dev_flagged) against the host producer: rows, KernelParams, fov, the table, its bounds,
  synchronous and enqueued calls;
- the device producer's trust verdict word against gf_table_flags_host of the same table, including tables built so that one block or
  one band of rows decides the word, and enough launches to wrap the pool of accumulator / ticket pairs;
- device tables and device verdicts straight into the packed warp kernel, against the oracle on the read-back tables."""
import numpy as np
import pytest

import gyroflow_b200 as g
from gyroflow_b200 import synth
from tests import cases, np_producer, producer_cases as pc

SENTINEL = -1                                  # 0xFFFFFFFF: a NaN no producer writes, and no verdict word either
ERR_BUFFER_TOO_SMALL = -7


def _case_ids():
    return sorted(pc.CASES)


# ------------------------------------------------------------------------------------------------ CPU: host producer vs numpy
@pytest.mark.parametrize("name", _case_ids())
def test_host_producer_matches_numpy_on_every_case(name):
    case = pc.CASES[name]
    org, sm = cases.gyro()
    p, cp, stab = pc.make(case, org, sm)
    for ts, frame in case["frames"]:
        kp, m, fov, _ = cp.at_timestamp(ts, frame)
        want, fov64 = pc.np_expected(case, p, org, sm, stab, ts, frame)
        assert m.shape == want.shape and kp.matrix_count == want.shape[0], (ts, frame)
        assert kp.fov == np.float32(fov64)
        assert pc.table_ulp_max(m[:, :9], want[:, :9]) <= 1.0, (ts, frame)
        assert float(pc.ulp_diff(m[:, 9:], want[:, 9:]).max()) <= 1.0, (ts, frame)
        if stab is not None and frame < len(stab) and "ibis" in stab[frame] and not (case.get("c", {}).get("suppress_rotation") and want.shape[0] == 1):
            assert np.abs(want[:, 9:]).max() > 0.0, (ts, frame)          # the IBIS columns really are exercised


def test_zero_shift_rule_and_stab_lookup_of_the_restatement():
    """The restatement's own edges: suppress_rotation without rolling shutter zeroes the shifts, with rolling shutter it keeps them;
    frames past the end of camera_stab have none; the scalar sync offset applies only without sync points."""
    org, sm = cases.gyro()
    p = synth.base_kernel_params(640, 360)
    stab = pc.spline_stab([12])
    on = np_producer.frame_matrices(p, org, sm, 900.0, suppress_rotation=True, camera_stab=stab)
    off = np_producer.frame_matrices(p, org, sm, 900.0, frame_readout_time_ms=0.0, suppress_rotation=True, camera_stab=stab)
    past = np_producer.frame_matrices(p, org, sm, 900.0, camera_stab=stab, frame=1)
    assert np.abs(on[:, 9:]).max() > 1.0 and (off[:, 9:] == 0).all() and (past[:, 9:] == 0).all()
    assert (on[:, :9] == on[0, :9]).all()                                # no rotation: every row is inverse(new_k)
    assert np_producer.offset_at_timestamp({}, 5.0, 6.5) == 6.5 and np_producer.offset_at_timestamp({1000: 2.0}, 5.0, 6.5) == 2.0


def test_null_spline_pointers_mean_no_points():
    """A camera_stab entry whose spline pointers are null has no points, whatever its count says: the host producer leaves those
    columns zero instead of reading through the null pointer (the device upload has always treated it so)."""
    case = pc.CASES["stab_null_pointers"]
    org, sm = cases.gyro()
    p, cp, stab = pc.make(case, org, sm)
    _, m0, _, _ = cp.at_timestamp(400.0, 0)          # IBIS pointer null, OIS present
    _, m2, _, _ = cp.at_timestamp(2300.0, 2)         # both null
    assert (m0[:, 9:12] == 0).all() and np.abs(m0[:, 12:]).max() > 0.1
    assert (m2[:, 9:] == 0).all()


# ------------------------------------------------------------------------------------------------ GPU helpers
def _buffers(torch, rows_alloc, n_words=1):
    tab = torch.empty((rows_alloc, 14), dtype=torch.int32, device="cuda")
    word = torch.empty(n_words, dtype=torch.int32, device="cuda")
    return tab, word


def _arm(torch, tab, word):
    tab.fill_(SENTINEL); word.fill_(SENTINEL)
    torch.cuda.synchronize()                       # the producer's stream is not torch's


def _read(tab, word, rows):
    t = tab.cpu().numpy()
    assert (t[rows:] == SENTINEL).all(), "rows at and after %d were written" % rows
    return t[:rows].view(np.float32).copy(), [int(v) & 0xFFFFFFFF for v in word.cpu().numpy()]


# ------------------------------------------------------------------------------------------------ GPU: device producer vs host producer
@pytest.mark.gpu
def test_device_producer_matches_host_on_every_case():
    import torch
    org, sm = cases.gyro()
    side = torch.cuda.Stream()
    n_cmp = n_words = 0
    same = total = 0
    worst = (2.0, "")
    for name in _case_ids():
        case = pc.CASES[name]
        p, cp, _ = pc.make(case, org, sm)
        dg = g.DeviceGyro(cp)
        rows_alloc = max(p.width, p.height) + 40
        tab, word = _buffers(torch, rows_alloc)
        case_same = case_total = 0
        for ts, frame in case["frames"]:
            kp_h, m_h, fov_h, mfov_h = cp.at_timestamp(ts, frame)
            _arm(torch, tab, word)
            kp, rows, fov, mfov = dg.frame_transform(ts, tab.data_ptr(), rows_alloc, frame=frame, table_flags_dev=word.data_ptr(), with_fov=True)
            assert rows == m_h.shape[0] and bytes(kp) == bytes(kp_h) and fov == fov_h and mfov == mfov_h, (name, ts, frame)
            got, (w,) = _read(tab, word, rows)
            s = pc.compare_tables(got, m_h)
            case_same += s; case_total += got[:, :9].size
            assert w == pc.table_flags_host(got), (name, ts, frame, w)
            # the same call enqueued on a side stream: identical table and word
            _arm(torch, tab, word)
            dg.frame_transform(ts, tab.data_ptr(), rows_alloc, frame=frame, table_flags_dev=word.data_ptr(), stream=side.cuda_stream)
            side.synchronize()
            got2, (w2,) = _read(tab, word, rows)
            assert np.array_equal(got2.view(np.uint32), got.view(np.uint32)) and w2 == w, (name, ts, frame)
            # one row short: an error before anything is enqueued, nothing written
            _arm(torch, tab, word)
            with pytest.raises(g.GyroflowCoreError) as e:
                dg.frame_transform(ts, tab.data_ptr(), rows - 1, frame=frame, table_flags_dev=word.data_ptr(), stream=side.cuda_stream)
            assert e.value.code == ERR_BUFFER_TOO_SMALL
            torch.cuda.synchronize()
            assert (tab.cpu().numpy() == SENTINEL).all() and int(word.cpu().numpy()[0]) == SENTINEL
            n_cmp += 1; n_words += 2
        dg.close()
        same += case_same; total += case_total
        worst = min(worst, (case_same / case_total, name))
    print("\ndevice producer vs host: %d (case, frame) comparisons over %d cases; columns 0-8 bit-identical: %.4f %% "
          "(lowest case %s: %.4f %%), largest difference %.1f ulp; %d verdict words checked"
          % (n_cmp, len(pc.CASES), 100.0 * same / total, worst[1], 100.0 * worst[0], pc.STATS["max_ulp"], n_words))
    assert worst[0] >= 0.99, worst


# ------------------------------------------------------------------------------------------------ GPU: engineered verdicts
TALL_W, TALL_H = 1024, 4320                        # 34 producer blocks, the last one partial (96 rows)
BIG_INDEX, WILD_TS, TAME_TS = 4000, 2006.0, 1000.0  # 2000 Hz track: sample 4000 is t = 2000 ms, 2 ms after the readout of WILD_TS starts


def _verdict_job(lens="opencv_fisheye", digital=None):
    """One 1024 x 4320 job whose (timestamp, frame) choices give all four verdicts.

    Frames 0, 1, 2 carry an IBIS band confined to one producer block: the first, block 17, the last (partial) one; frame 3 is past
    the end of camera_stab.  The org track's sample BIG_INDEX is scaled by 1e7 (not a unit quaternion), so the rows whose lookup lands
    on [t_k, t_k+1) get entries below 2^-40: WILD_TS has wild rows in one band near the start of its readout, TAME_TS has none.
    (A NaN sample would not do: the cofactor inverse of a NaN matrix is the zero matrix, which is tame.)"""
    org, sm = synth.synthetic_gyro(4.0, rate_hz=2000.0)
    org = synth.GyroTrack(org.ts.copy(), org.q.copy())
    org.q[BIG_INDEX] *= 1e7
    blocks = [0, 17, 33]
    rows = [(b * pc.BLOCK + 12, min(b * pc.BLOCK + 110, TALL_H - 4)) for b in blocks]
    stab = pc.spline_stab([10, 13, 8], ois=False, band=[pc.band_for_rows(TALL_H, r0, r1) for r0, r1 in rows])
    p = synth.base_kernel_params(TALL_W, TALL_H, lens=lens, digital_lens=digital)
    cp = g.ComputeParams(p, org, sm, camera_stab=stab)
    choices = {0: (TAME_TS, 3), 1: (WILD_TS, 3), 2: (TAME_TS, 0), 3: (WILD_TS, 0)}
    return p, cp, blocks, choices


def _blocks_of(mask):
    return sorted(set((np.nonzero(mask)[0] // pc.BLOCK).tolist()))


@pytest.mark.gpu
def test_verdict_word_on_engineered_tables():
    import torch
    p, cp, _, choices = _verdict_job()
    dg = g.DeviceGyro(cp)
    tab, word = _buffers(torch, TALL_H + 40)
    n = 0
    for ts, frame, want_word, want_ibis_block in [(TAME_TS, 0, 2, 0), (TAME_TS, 1, 2, 17), (TAME_TS, 2, 2, 33), (WILD_TS, 3, 1, None),
                                                  (WILD_TS, 0, 3, 0), (WILD_TS, 2, 3, 33), (TAME_TS, 3, 0, None)]:
        _arm(torch, tab, word)
        kp, rows = dg.frame_transform(ts, tab.data_ptr(), TALL_H + 40, frame=frame, table_flags_dev=word.data_ptr())
        got, (w,) = _read(tab, word, rows)
        assert rows == TALL_H and w == pc.table_flags_host(got) == want_word, (ts, frame, w)
        ibis_rows = (got[:, 9:] != 0).any(axis=1)
        wild_rows = np.array([pc.table_flags_host(got[r:r + 1]) & 1 for r in range(rows)], bool) if want_word & 1 else np.zeros(rows, bool)
        assert _blocks_of(ibis_rows) == ([want_ibis_block] if want_ibis_block is not None else [])
        if want_word & 1:
            wb = _blocks_of(wild_rows)
            assert 0 < len(wb) <= 2 and wb[0] >= 2 and wb[-1] <= 6, wb       # one band near the start of the readout
        pc.compare_tables(got, cp.at_timestamp(ts, frame)[1])
        n += 1
    # a one-row table (readout time 0): the single row decides the word
    p1 = synth.base_kernel_params(640, 360)
    org, sm = cases.gyro()
    for stab, want_word in ((None, 0), (pc.spline_stab([12]), 2)):
        cp1 = g.ComputeParams(p1, org, sm, frame_readout_time_ms=0.0, camera_stab=stab)
        dg1 = g.DeviceGyro(cp1)
        t1, w1 = _buffers(torch, 8)
        _arm(torch, t1, w1)
        _, rows = dg1.frame_transform(900.0, t1.data_ptr(), 8, table_flags_dev=w1.data_ptr())
        got, (w,) = _read(t1, w1, rows)
        assert rows == 1 and w == pc.table_flags_host(got) == want_word
        dg1.close(); n += 1
    dg.close()
    print("\nengineered verdicts: %d verdict words checked" % n)


@pytest.mark.gpu
def test_verdict_word_when_the_last_block_runs_waves_after_the_first():
    """A horizontal-readout table of 2^19 rows is 4096 producer blocks, several waves of an H100 (at most 9 blocks of 128 threads
    per SM at 54 registers): its only IBIS rows are in the last block, which runs long after block 0 has finished.  The word is still
    2, because the last block to finish publishes it; a frame without camera_stab gives 0 with the same accumulator pool."""
    import torch
    w, h = 1 << 19, 360
    last = w // pc.BLOCK - 1
    stab = pc.spline_stab([9], ois=False, band=[pc.band_for_rows(h, last * pc.BLOCK + 10, last * pc.BLOCK + 100)])
    org, sm = cases.gyro()
    cp = g.ComputeParams(synth.base_kernel_params(w, h), org, sm, horizontal=True, camera_stab=stab)
    dg = g.DeviceGyro(cp)
    tab, word = _buffers(torch, w + 8)
    for frame, want_word in ((0, 2), (1, 0), (0, 2), (1, 0)):
        _arm(torch, tab, word)
        _, rows = dg.frame_transform(1500.0, tab.data_ptr(), w + 8, frame=frame, table_flags_dev=word.data_ptr())
        got, (wd,) = _read(tab, word, rows)
        assert rows == w and wd == pc.table_flags_host(got) == want_word, (frame, wd)
        assert _blocks_of((got[:, 9:] != 0).any(axis=1)) == ([last] if want_word else [])
    pc.compare_tables(got, cp.at_timestamp(1500.0, 1)[1])
    dg.close()
    print("\nmulti-wave table: 4 verdict words checked")


@pytest.mark.gpu
def test_verdict_word_rearms_across_streams_and_pool_wrap():
    """One DeviceGyro, 72 launches cycling through the four verdicts on three streams (each with its own table) and no host sync inside a
    window of 12 launches: every launch's word equals the host scan of its table.  72 > 64 accumulator / ticket pairs, so the pool
    wraps, and the pairs it reuses produce a different word the second time."""
    import torch
    p, cp, _, choices = _verdict_job()
    dg = g.DeviceGyro(cp)
    rows_alloc = TALL_H + 40
    want = {}
    tab, word = _buffers(torch, rows_alloc)
    for v, (ts, frame) in choices.items():                   # the word each choice must give, from its read-back table
        _arm(torch, tab, word)
        _, rows = dg.frame_transform(ts, tab.data_ptr(), rows_alloc, frame=frame, table_flags_dev=word.data_ptr())
        got, (w,) = _read(tab, word, rows)
        assert pc.table_flags_host(got) == v == w
        want[v] = got
    streams = [torch.cuda.Stream() for _ in range(3)]
    tabs = [torch.empty((rows_alloc, 14), dtype=torch.int32, device="cuda") for _ in streams]
    n_launch, window = 72, 12
    words = torch.full((n_launch,), SENTINEL, dtype=torch.int32, device="cuda")
    # every verdict on every stream; neighbours on one stream differ, and so do launch i and launch i + 64, which share a pair
    order = [(i * 3 + i // 4 + i // 64) % 4 for i in range(n_launch)]
    checked = 0
    for base in range(0, n_launch, window):
        for t in tabs: t.fill_(SENTINEL)
        torch.cuda.synchronize()
        for i in range(base, base + window):
            ts, frame = choices[order[i]]
            dg.frame_transform(ts, tabs[i % 3].data_ptr(), rows_alloc, frame=frame, table_flags_dev=words[i:].data_ptr(), stream=streams[i % 3].cuda_stream)
        torch.cuda.synchronize()
        for k in range(3):                                   # each stream's table is its last launch's
            last = max(i for i in range(base, base + window) if i % 3 == k)
            got = tabs[k].cpu().numpy()[:TALL_H].view(np.float32)
            assert np.array_equal(got.view(np.uint32), want[order[last]].view(np.uint32)), (last, order[last])
    got_words = [int(v) & 0xFFFFFFFF for v in words.cpu().numpy()]
    assert got_words == order, [(i, a, b) for i, (a, b) in enumerate(zip(got_words, order)) if a != b][:8]
    checked += len(got_words)
    dg.close()
    print("\nre-arm / pool wrap: %d verdict words checked over 3 streams" % checked)


# ------------------------------------------------------------------------------------------------ GPU: device table + verdict -> packed kernel
@pytest.mark.gpu
@pytest.mark.parametrize("lens,digital", [("opencv_fisheye", None), ("poly3", None), ("sony", "digital_stretch")])
def test_device_tables_and_verdicts_into_the_packed_kernel(lens, digital):
    """Producer and warp on one stream, no host sync between them, the warp reading the producer's verdict word: bytes == the oracle
    on the read-back table.  A word that wrongly said 0 for the IBIS band or the wild band would send that table down the trusted path,
    which skips the per-pixel IBIS and numerator tests."""
    import torch
    from tests import oracle_lib
    pix = "RGBA8"
    _, cp, _, choices = _verdict_job(lens, digital)
    p = synth.base_kernel_params(TALL_W, TALL_H, pixel_type=pix, lens=lens, digital_lens=digital)
    dg = g.DeviceGyro(cp)
    st = g.stab_config(p, pix, digital_lens=digital)
    src = synth.synthetic_frame(TALL_W, TALL_H, pix, stride=p.stride)
    tsrc = torch.from_numpy(src).cuda()
    tdst = torch.zeros((TALL_H, p.output_stride), dtype=torch.uint8, device="cuda")
    bufs = g.Buffers(g.BufferDescription((TALL_W, TALL_H, p.stride), tsrc.data_ptr(), length=tsrc.numel()),
                     g.BufferDescription((TALL_W, TALL_H, p.output_stride), tdst.data_ptr(), length=tdst.numel()))
    wr = g.CudaWrapper.new(p, pix, lens, digital, bufs)
    tab, word = _buffers(torch, TALL_H)
    side = torch.cuda.Stream()
    for v, (ts, frame) in sorted(choices.items()):
        _arm(torch, tab, word); tdst.fill_(0); torch.cuda.synchronize()
        kp, rows = dg.frame_transform(ts, tab.data_ptr(), TALL_H, frame=frame, table_flags_dev=word.data_ptr(), stream=side.cuda_stream)
        kp = g.get_frame_transform_at(st, cp, bufs, kp, frame=frame)
        wr.undistort_image_dev(bufs, kp, tab.data_ptr(), rows, stream=side.cuda_stream, table_flags_dev=word.data_ptr())
        side.synchronize()
        got, (w,) = _read(tab, word, rows)
        assert w == v == pc.table_flags_host(got)
        ref = np.zeros((TALL_H, p.output_stride), np.uint8)
        assert oracle_lib.undistort_image(src, ref, kp, pix, lens, digital, got) == 0
        out = tdst.cpu().numpy()
        bad = np.nonzero(out != ref)
        assert bad[0].size == 0, "verdict %d: %d bytes differ, first at row %d" % (v, bad[0].size, int(bad[0][0]))
    wr.close(); dg.close()
