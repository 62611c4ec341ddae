"""CPU emulation of the packed warp kernel's 8-bit interior sampler (warp_kernel_x2.cuh: hot_w, hot_interior, sample_u8_hot).

The kernel's integer arithmetic is replayed with numpy in 32-bit wrapping words and compared with what the scalar kernels compute:
  * the biased rounding word: bits(RZ(64 u + 2^23)) - (0x4affffff + 64 rx0) against round_half_away_w(64 u) - 64 rx0, and the
    interior test `(unsigned) w' <= 64 span + 63` against `(unsigned)((w >> 6) - rx0) <= span`;
  * the doubled weights: w & 62 == 2 fx, 64 + 255 * (2 fy) holds the bytes (64 - 2 fy, 2 fy), and the 16-bit-lane blend with dp2a
    gives 4 N, so that 4 N >> 12 == N >> 10 with N = sum p * wx * wy (sample_u8_bilinear).
"""
import numpy as np

U32 = np.uint32


def _rz_add_2p23(a2):
    """RZ(a2 + 2^23) for float32 a2 with 0 <= a2 + 2^23 < 2^24 (exact sum in float64, then truncation to the float32 grid)."""
    s = a2.astype(np.float64) + 8388608.0
    out = np.empty_like(s)
    hi = s >= 8388608.0                          # spacing 1 in [2^23, 2^24)
    out[hi] = np.floor(s[hi])
    out[~hi] = np.floor(s[~hi] * 2.0) / 2.0      # spacing 1/2 in [2^22, 2^23)
    return out.astype(np.float32)


def _bits(f):
    return f.view(np.int32).astype(np.int64)


def test_biased_word_and_interior_test():
    rng = np.random.default_rng(11)
    for rx0, span in ((0, 3838), (1, 100), (37, 2000), (65535 - 300, 290)):
        # every 1/128 of a pixel across the rect and beyond both edges, plus random values
        u = np.concatenate([np.arange(-3.0, rx0 + span + 4.0, 1.0 / 128.0) + (rx0 - 2.0 if rx0 else 0.0),
                            rng.uniform(-10.0, rx0 + span + 10.0, 20000)]).astype(np.float32)
        u = u[np.abs(u) < 65536.0]
        s = _rz_add_2p23(u * np.float32(64.0))
        w = _bits(s) - 0x4affffff                                        # round_half_away_w
        wb = _bits(s) - (0x4affffff + 64 * rx0)                          # hot_w
        assert np.array_equal(wb, w - 64 * rx0)
        old = ((w >> 6) - rx0).astype(np.int64) & 0xffffffff <= span
        new = (wb & 0xffffffff) <= 64 * span + 63
        assert np.array_equal(old, new)
        # inside, the word gives the same column and fraction as the unbiased one
        assert np.array_equal((wb[new] >> 6) + rx0, w[new] >> 6)
        assert np.array_equal(wb[new] & 62, 2 * ((w[new] >> 1) & 31))


def _dp2a_lo(a, b):
    return ((a & 0xffff) * (b & 0xff) + (a >> 16) * ((b >> 8) & 0xff)) & 0xffffffff


def _perm_lo(x, y):      # __byte_perm(x, y, 0x5410): x.lo16 | y.lo16 << 16
    return (x & 0xffff) | ((y & 0xffff) << 16)


def _perm_hi(x, y):      # __byte_perm(x, y, 0x7632): x.hi16 | y.hi16 << 16
    return (x >> 16) | (y & 0xffff0000)


def _odd(p):             # __byte_perm(p, 0, 0x4341): byte 1 | byte 3 << 16
    return ((p >> 8) & 0xff) | (((p >> 24) & 0xff) << 16)


def test_doubled_weight_blend_matches_integer_bilinear():
    rng = np.random.default_rng(5)
    n = 200000
    taps = rng.integers(0, 256, size=(n, 4, 4), dtype=np.int64)         # p00, p01, p10, p11 x RGBA
    taps[:1000] = 255                                                    # the largest lane values
    taps[1000:2000] = 0
    fx = rng.integers(0, 32, size=n, dtype=np.int64)
    fy = rng.integers(0, 32, size=n, dtype=np.int64)
    fx[:64] = np.arange(64) % 32; fy[:64] = np.arange(64) // 2 % 32
    word = lambda t: t[:, 0] | (t[:, 1] << 8) | (t[:, 2] << 16) | (t[:, 3] << 24)
    p00, p01, p10, p11 = (word(taps[:, i]) for i in range(4))
    fx2, fy2 = 2 * fx, 2 * fy
    wx0, wx1 = 64 - fx2, fx2
    wy = 64 + 255 * fy2
    assert np.all((wy & 0xff) == 64 - fy2) and np.all((wy >> 8) == fy2)
    m = lambda v: v & 0xffffffff
    he0 = m((p00 & 0x00ff00ff) * wx0 + (p01 & 0x00ff00ff) * wx1)
    he1 = m((p10 & 0x00ff00ff) * wx0 + (p11 & 0x00ff00ff) * wx1)
    ho0 = m(_odd(p00) * wx0 + _odd(p01) * wx1)
    ho1 = m(_odd(p10) * wx0 + _odd(p11) * wx1)
    got = [_dp2a_lo(_perm_lo(he0, he1), wy) >> 12, _dp2a_lo(_perm_lo(ho0, ho1), wy) >> 12,
           _dp2a_lo(_perm_hi(he0, he1), wy) >> 12, _dp2a_lo(_perm_hi(ho0, ho1), wy) >> 12]
    for ch in range(4):
        N = (taps[:, 0, ch] * (32 - fx) + taps[:, 1, ch] * fx) * (32 - fy) + (taps[:, 2, ch] * (32 - fx) + taps[:, 3, ch] * fx) * fy
        assert np.array_equal(got[ch], N >> 10), ch
