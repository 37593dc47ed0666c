"""Numerical model (numpy, CPU) of the error-compensated fp16 split the default conv math mode uses on the tensor cores
(3d-sis_b200/csrc/conv_tc.cu: split_f16, the X3 = 2 kernels; DESIGN.md §4.1).  v = hi + lo / 2048 with hi = fp16(v),
lo = fp16((v - hi) * 2048); a product a*b is ah*bh + (ah*bl + al*bh) / 2048 with fp32 accumulation, the al*bl term dropped.
The properties below are what the 'exact' mode's parity claim (integer outputs equal to the fp32 path) rests on; the kernels
themselves are checked on the GPU (tests/test_gpu_tc_accuracy.py, tests/test_gpu_forward.py)."""
import numpy as np


def split(v):
    v = np.clip(v.astype(np.float32), -65504, 65504)
    hi = v.astype(np.float16)
    lo = ((v - hi.astype(np.float32)) * np.float32(2048)).astype(np.float16)
    return hi, lo


def test_split_keeps_22_significand_bits_over_the_fp16_normal_range():
    rng = np.random.default_rng(0)
    v = (rng.choice([-1.0, 1.0], 200000) * np.exp(rng.uniform(np.log(1e-4), np.log(6e4), 200000))).astype(np.float32)
    hi, lo = split(v)
    assert np.isfinite(hi.astype(np.float32)).all() and np.isfinite(lo.astype(np.float32)).all()
    rec = hi.astype(np.float64) + lo.astype(np.float64) / 2048
    rel = np.abs(rec - v.astype(np.float64)) / np.abs(v.astype(np.float64))
    assert rel.max() <= 2.0 ** -22
    # without the 2048 scale the low part of an O(1e-2) value would be an fp16 SUBNORMAL (|v - hi| <= 2^-11 |v| < 6.1e-5) and lose
    # bits; scaled, it is a normal number except when v happens to lie within 1 % of an fp16 value
    big = (np.abs(v) >= 1e-2) & (lo != 0)
    assert (np.abs(lo[big].astype(np.float32)) >= 2.0 ** -14).mean() > 0.99
    assert (np.abs(v[big] - hi[big].astype(np.float32)) < 2.0 ** -14).mean() > 0.2


def test_small_magnitudes_degrade_gracefully_in_absolute_terms():
    """Below fp16's normal range (|v| < 6.1e-5) hi is subnormal; the absolute error stays below 2^-35, i.e. far under the fp32
    rounding error of any sum it is added to with O(1e-3 .. 1) terms (activations after ReLU, BN-folded weights)."""
    rng = np.random.default_rng(1)
    v = (rng.standard_normal(100000) * 10.0 ** rng.uniform(-9, -4.3, 100000)).astype(np.float32)
    hi, lo = split(v)
    rec = hi.astype(np.float64) + lo.astype(np.float64) / 2048
    assert np.abs(rec - v.astype(np.float64)).max() <= 2.0 ** -35


def test_three_products_match_fp32_dot_products_of_conv_length():
    """K = 27 taps x 64 channels.  ah*bh, ah*bl and al*bh are exact in fp32 (11 x 11 significand bits); what is lost is al*bl
    (<= 2^-22 relative per term) and the accumulation rounding, which the fp32 CUDA-core path has too."""
    rng = np.random.default_rng(2)
    K, N = 27 * 64, 4000
    a = np.maximum(rng.standard_normal((N, K)), 0).astype(np.float32)          # post-ReLU activations
    b = (rng.standard_normal((N, K)) * 0.05).astype(np.float32)                # weights
    ah, al = split(a)
    bh, bl = split(b)
    f32 = lambda x: x.astype(np.float32)
    main = np.zeros(N, np.float32)
    cross = np.zeros(N, np.float32)
    for k0 in range(0, K, 32):                                                  # one MMA = 32 K-elements, summed into fp32
        s = slice(k0, k0 + 32)
        main += (f32(ah[:, s]).astype(np.float64) * f32(bh[:, s])).sum(1).astype(np.float32)
        cross += (f32(ah[:, s]).astype(np.float64) * f32(bl[:, s]) + f32(al[:, s]).astype(np.float64) * f32(bh[:, s])).sum(1).astype(np.float32)
    got = main + cross * np.float32(1.0 / 2048)
    ref64 = (a.astype(np.float64) * b.astype(np.float64)).sum(1)
    ref32 = np.zeros(N, np.float32)
    for k in range(K):                                                          # a plain fp32 chain, like one CUDA-core thread
        ref32 += a[:, k] * b[:, k]
    scale = (np.abs(a.astype(np.float64)) * np.abs(b.astype(np.float64))).sum(1)
    err_split = np.abs(got - ref64) / scale
    err_fp32 = np.abs(ref32 - ref64) / scale
    assert err_split.max() <= 2.0 ** -21                                       # 22-bit operands + fp32 sums
    assert err_split.mean() <= err_fp32.mean()                                  # blocked sums beat the serial fp32 chain
    # the plain fp16-operand product (what the 'fp16' mode computes) is three orders of magnitude coarser
    err_fp16 = np.abs((f32(ah).astype(np.float64) * f32(bh)).sum(1) - ref64) / scale
    assert err_fp16.mean() > 200 * err_split.mean()


def test_dropped_low_low_term_is_below_the_operand_precision():
    rng = np.random.default_rng(3)
    mag = lambda: (rng.choice([-1.0, 1.0], 100000) * np.exp(rng.uniform(np.log(1e-3), np.log(1e3), 100000))).astype(np.float32)
    a, b = mag(), mag()
    ah, al = split(a)
    bh, bl = split(b)
    dropped = np.abs(al.astype(np.float64) * bl.astype(np.float64)) / 2048 ** 2
    assert (dropped / np.abs(a.astype(np.float64) * b.astype(np.float64))).max() <= 2.0 ** -22


def _stage_model(a, b, drop=None):
    """The X3 = 2 main loop per output element: operands split as split_f16; each 16-element MMA summed exactly and added to
    the stage's fresh accumulator with truncation toward zero; a stage (3 x-taps x 32 channels = 96 K-elements) folded into
    the running sum as fmaf(cross, 2^-11, sum) (round to nearest), then its hi.hi part.  drop: "cross" (no cross terms, the
    1x product), "albh" (one cross term), or a stage index whose cross terms are lost."""
    def parts(v):
        hi, lo = split(v)
        return hi.astype(np.float64), lo.astype(np.float64)

    def trunc_add(acc, t):
        s = acc.astype(np.float64) + t
        r = s.astype(np.float32)
        over = np.abs(r.astype(np.float64)) > np.abs(s)
        r[over] = np.nextafter(r[over], np.float32(0))
        return r

    (ah, al), (bh, bl) = parts(a), parts(b)
    acc = np.zeros(a.shape[0], np.float32)
    for st in range(a.shape[1] // 96):
        cross = np.zeros_like(acc)
        hh = np.zeros_like(acc)
        for m in range(6):
            s = slice(st * 96 + m * 16, st * 96 + m * 16 + 16)
            if drop not in ("cross", st):
                if drop != "albh":
                    cross = trunc_add(cross, (al[:, s] * bh[:, s]).sum(1))
                cross = trunc_add(cross, (ah[:, s] * bl[:, s]).sum(1))
            hh = trunc_add(hh, (ah[:, s] * bh[:, s]).sum(1))
        acc = (cross.astype(np.float64) * 2.0 ** -11 + acc.astype(np.float64)).astype(np.float32)
        acc = (acc.astype(np.float64) + hh).astype(np.float32)
    return acc


def test_per_element_bound_separates_the_compensated_kernel_from_broken_ones():
    """The bound of tests/test_gpu_tc_accuracy.py, |err| <= C_X3 s2 + C_T |ref| with s2 = sqrt(sum_k (x_k w_k)^2), holds for the
    modelled kernel and is exceeded at least POWER-fold by each model of a kernel that lost (part of) the compensation, at
    K = 27 * 32 and 27 * 256.  Keeps the GPU test's constants honest without a GPU."""
    from test_gpu_tc_accuracy import C_T, C_X3, POWER
    rng = np.random.default_rng(4)
    for K in (864, 6912):
        a = np.maximum(rng.standard_normal((2000, K)), 0).astype(np.float32)  # post-ReLU activations
        b = (rng.standard_normal((2000, K)) / np.sqrt(K)).astype(np.float32)  # weights N(0, 1/K)
        p = a.astype(np.float64) * b.astype(np.float64)
        ref = p.sum(1)
        bound = C_X3 * np.sqrt((p * p).sum(1)) + C_T * np.abs(ref)
        ratio = lambda drop: (np.abs(_stage_model(a, b, drop).astype(np.float64) - ref) / bound).max()
        assert ratio(None) <= 1.0, (K, ratio(None))
        for drop in ("cross", "albh", K // 96 - 1):
            assert ratio(drop) >= POWER, (K, drop, ratio(drop))
