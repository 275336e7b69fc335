"""CPU check of the EXACT_TC error model (oracle/split_operands.py): the three-term split-fp16 product is as good as an
fp32 GEMM when the weight planes are scaled into the normal fp16 range, and measurably worse when they are not (conv1's
BN-folded weights are ~1e-3: their `lo` plane would be subnormal)."""
import torch

from oracle import split_operands as S


def rel(a, ref):
    return float((a.double() - ref).norm() / ref.norm())


def gemm(seed, M, K, N, w_scale):
    g = torch.Generator().manual_seed(seed)
    a = torch.relu(torch.randn(M, K, generator=g)) * 3.0          # post-ReLU activations
    b = torch.randn(K, N, generator=g) * w_scale
    return a, b, a.double() @ b.double()


def test_split_product_matches_fp32_when_weights_are_scaled():
    for seed, w_scale in ((1, 1.0e-3), (2, 5.0e-2), (3, 2.0)):
        a, b, ref = gemm(seed, 256, 576, 96, w_scale)
        e32 = rel(a @ b, ref)
        e_split = rel(S.split_matmul(a, b), ref)
        e16 = rel(S.fp16_matmul(a, b), ref)
        assert e_split < 1.0e-6 and e_split < 4.0 * e32 + 1.0e-7, (w_scale, e_split, e32)
        assert e16 > 50.0 * e_split, (w_scale, e16, e_split)       # plain fp16 operands: ~3e-4


def test_unscaled_small_weights_lose_the_lo_plane():
    a, b, ref = gemm(4, 256, 147, 64, 1.0e-3)                       # conv1-like: 7x7x3 taps, folded weights ~1e-3
    e_scaled = rel(S.split_matmul(a, b, scale_weights=True), ref)
    e_unscaled = rel(S.split_matmul(a, b, scale_weights=False), ref)
    assert e_scaled < 1.0e-6
    assert e_unscaled > 10.0 * e_scaled, (e_unscaled, e_scaled)


def test_weight_scale_is_a_power_of_two_into_the_target_range():
    for m in (1.0e-4, 3.3e-3, 0.7, 1.0, 5000.0, 8192.0):
        s = S.weight_scale(torch.tensor([m, -m / 3]))
        assert 4096.0 <= m * s < 8192.0
        mant, _ = __import__("math").frexp(s)
        assert mant == 0.5                                          # exact power of two: scaling loses no bits
    assert S.weight_scale(torch.zeros(3)) == 1.0


def test_dropped_lo_lo_term_is_below_fp32_rounding():
    a, b, ref = gemm(5, 128, 1152, 128, 2.0e-2)
    s = S.weight_scale(b)
    a_hi, a_lo = S.split(a)
    b_hi, b_lo = S.split(b * s)
    three = (a_lo.double() @ b_hi.double() + a_hi.double() @ b_lo.double() + a_hi.double() @ b_hi.double()) / s
    four = three + (a_lo.double() @ b_lo.double()) / s
    assert rel(three.float(), ref) < 5.0e-7
    assert abs(rel(four.float(), ref) - rel(three.float(), ref)) < 5.0e-8


# ---- gradient planes ---------------------------------------------------------------------------------------------------------
def test_grad_exponent_brings_the_entry_gradient_into_its_window():
    lo, hi = 2.0 ** (S.GRAD_EXP_TOP - 1), 2.0 ** S.GRAD_EXP_TOP
    for amax in (4.2e-4, 1.8e-5, 0.04, 3.0, 7.0e4, 1e-20, 2.0 ** -20, 49.0 / 4096 * 2 ** 7):
        for gs in (1.0, 4096.0, 1000.0, 2.0 ** 20):
            k = S.grad_exponent(amax, gs)
            assert lo <= amax * gs * 2.0 ** k / 49 < hi, (amax, gs, k)
    assert S.grad_exponent(0.0, 4096.0) == 0
    assert S.grad_exponent(float("nan"), 4096.0) == 0 and S.grad_exponent(float("inf"), 1.0) == 0
    assert S.grad_exponent(1e-44, 1.0) == S.GRAD_EXP_MAX and S.grad_exponent(3e38, 2.0 ** 60) == -S.GRAD_EXP_MAX


def test_step_gradient_split_error():
    """the gradient one SSN training step hands the backbone (oracle step_check.ssn_step_dfeat; one frame through the synthetic
    backbone in float64, its gradient that of the first frame of an incomplete proposal, which only the completeness loss
    reaches: max |dfeat| 1.1e-5, the step's median magnitude): the fp16 planes of every convolution output's dz * grad_scale lose bits at bench.py's grad_scale
    4096 (lo is subnormal below 2^-3, hi below 2^-14) and flush most of it at grad_scale 1; with the exponent rule both carry
    the fp32 gradient to the split's 22 bits"""
    from oracle import ssn_oracle as O
    from oracle import step_check as SC
    from oracle import synth
    bb = {k: v.double() for k, v in synth.synth_backbone(3, seed=0, calib_frames=2).items()}
    x = synth.synth_frames(1, 3, seed=17).double().requires_grad_(True)
    taps = {}
    with torch.enable_grad():
        feat = O.backbone_forward(bb, x, 3, taps=taps)
        dfeat = SC.ssn_step_dfeat(feat.float().repeat(SC.STEP_PROPS * SC.STEP_SEG, 1))[SC.STEP_SEG:SC.STEP_SEG + 1].double()
        outs = [id_ + "_bn" for (id_, *_r) in O.conv_layers(3)]
        grads = torch.autograd.grad(feat, [taps[o] for o in outs], dfeat)
    dz = [(g * (taps[o] > 0)).float() for o, g in zip(outs, grads)]
    amax = float(dfeat.float().abs().max())
    err = {}
    for label, gs in (("4096", 4096.0), ("1", 1.0), ("rule 4096", 4096.0 * 2.0 ** S.grad_exponent(amax, 4096.0)),
                      ("rule 1", 2.0 ** S.grad_exponent(amax, 1.0))):
        err[label] = [S.split_error(d, gs) for d in dz]
    worst = {k: max(v) for k, v in err.items()}
    print("\nsplit error of dz, worst of 69 layers: %s; above 1.5e-5 at grad_scale 4096: %d layers"
          % (worst, sum(e > 1.5e-5 for e in err["4096"])))
    assert worst["4096"] > 1.5e-5 and worst["1"] > 1e-2
    assert worst["rule 4096"] <= 3e-7 and worst["rule 1"] <= 3e-7
