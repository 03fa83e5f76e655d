"""cutie_conv_tc (csrc/conv_tc.cu): the wgmma 3xTF32 implicit-GEMM 3x3 / 1x1 convolution against F.conv2d evaluated in
float64 (the ground truth) and against cuDNN's fp32 result (the library call it replaces): its error vs float64 must be of
the same class as cuDNN's own fp32 error -- never a TF32-class (1e-3 relative) one.

Every output element is also held to a bar of its own (_elementwise_err): its error over the float64 sum of the magnitudes
of the terms it adds up.  That bar does not depend on cuDNN.  The norm-wise bar does: its fixed 6e-5 cap alone passes a
defect confined to one 32-channel input chunk of a 512- or 1024-channel layer (test_per_element_bar_rejects_lo_term_defects)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method='thread')]

U = 2.0 ** -24                   # fp32 unit roundoff
# Largest per-element error r allowed (_elementwise_err), in units of U.  Measured on an H100 80GB HBM3 (400 W) over every
# case of this file and tests/test_gpu_conv_tc_f16.py: the 3xTF32 kernel reaches 7.53 U (1x1 64->256 at 120x216), the FP16
# one 2.89 U against its rounded operands.  The lo-term defects of test_per_element_bar_rejects_lo_term_defects score
# 124.7-2956 U; the weakest is one 32-channel chunk of the 3x3 512->768 layer (1/144 of K).  A 3xTF32 bar 4x above the
# kernel and 4x below every defect must lie in [30.1, 31.2] U, so both margins are thin (4.1x and 4.0x): a kernel change
# that raises the worst r above 7.75 U, or a larger-K layer in the defect list, leaves no such bar (the kernel's worst r
# is at small K, a one-chunk defect's r falls as K grows).
BAR_TF32 = 31 * U
BAR_F16 = 12 * U


def tf32_rna(t: torch.Tensor) -> torch.Tensor:
    """cvt.rna.tf32.f32 for finite and infinite fp32 values: keep 10 explicit mantissa bits, rounding to nearest with ties
    away from zero (add half a tf32 ulp to the magnitude, truncate; a carry moves into the exponent, so values within half
    a tf32 ulp of FLT_MAX round to inf).  Subnormals round the same way."""
    b = t.float().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b & 0x80000000) | (((b & 0x7FFFFFFF) + 0x1000) & 0x7FFFE000)
    return (r - ((r >> 31) << 32)).to(torch.int32).view(torch.float32).reshape(t.shape)


def _elementwise_err(got, x, w, b, z=None, relu_in=False, relu_out=False, stride=1, f16=False):
    """max over the output of r = |got - y64| / D: y64 = act(conv(pre(x), w) + b [+ z]) and D = conv(|pre(x)|, |w|) + |b|
    [+ |z|], both in float64 -- each element's error against the magnitude of the terms it sums, whatever their
    cancellation.  f16: the operands are the kernel's, pre(x) and w rounded to fp16 (b and z exact), so r is the
    accumulation error alone.  Where D == 0 every term is zero, and the output must be exactly zero."""
    pad = w.shape[-1] // 2
    pre = x.relu() if relu_in else x
    if f16:
        pre, w = pre.half().float(), w.half().float()
    pre, w = pre.double(), w.double()
    bd = b.double() if b is not None else None
    y = F.conv2d(pre, w, bd, stride=stride, padding=pad)
    D = F.conv2d(pre.abs(), w.abs(), bd.abs() if bd is not None else None, stride=stride, padding=pad)
    if z is not None:
        y, D = y + z.double(), D + z.double().abs()
    if relu_out:
        y = y.relu()
    assert got.shape == y.shape and got.dtype == torch.float32
    zero = D == 0
    assert bool((got[zero] == 0).all()), 'an output whose terms are all zero is not zero'
    return float(torch.where(zero, 0.0, (got.double() - y).abs() / D).max())


def _ref64(x, w, b, z, relu_in, relu_out):
    xx = x.double()
    if relu_in:
        xx = xx.relu()
    y = F.conv2d(xx, w.double(), b.double() if b is not None else None, padding=1)
    if z is not None:
        y = y + z.double()
    return y.relu() if relu_out else y


CASES = [
    # NB, Cin, Cout, H, W
    (3, 256, 256, 30, 54),        # PixelFFN / CAResBlock at 480p, 3 objects (cfg 2)
    (1, 256, 256, 30, 54),
    (2, 32, 128, 5, 7),           # one chunk, tiny image: every position near a border
    (1, 64, 128, 1, 1),
    (1, 96, 256, 17, 130),        # wider than one tile row: column tiles with halos
    (2, 128, 128, 60, 108),       # decoder shapes
    (1, 128, 128, 120, 216),
    (1, 512, 256, 23, 40),        # 16 chunks
    (1, 64, 64, 40, 72),          # half a channel tile (zero-padded weight rows)
    (3, 512, 768, 30, 54),        # sensory update: 6 channel tiles
    (1, 32, 200, 9, 9),           # ragged channel count
    (1, 64, 128, 1, 300),         # a single row: every tap row but the centre one reads padding
    (1, 64, 128, 300, 1),         # a single column
    (1, 64, 128, 30, 57),         # the widest whole-row tile at H = 30 (2 x 57, N = 128) ...
    (1, 64, 128, 30, 58),         # ... and one column more: two column tiles per row (3 x 29, N = 96)
    (40, 256, 256, 30, 54),       # 40 object images in one call (NB = B x objects is unbounded)
]


@pytest.mark.parametrize('NB,Cin,Cout,H,W', CASES)
@pytest.mark.parametrize('epi', ['plain', 'relu_in+residual', 'relu_out', 'no_bias'])
def test_conv3x3_tc_is_fp32_class_accurate(NB, Cin, Cout, H, W, epi):
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device='cuda').manual_seed(NB * 1000 + Cin + H)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g) * 1.5
    w = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) * (2.0 / (9 * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    z = torch.randn(NB, Cout, H, W, device='cuda', generator=g) if 'residual' in epi else None
    if epi == 'no_bias':
        b = None
    relu_in, relu_out = 'relu_in' in epi, 'relu_out' in epi
    img = K_.conv_weight_image(w)
    got = K_.conv_tc(x, img, b, Cout, residual=z, relu_in=relu_in, relu_out=relu_out)
    ref = _ref64(x, w, b, z, relu_in, relu_out)
    lib32 = F.conv2d(x.relu() if relu_in else x, w, b, padding=1)
    if z is not None:
        lib32 = lib32 + z
    if relu_out:
        lib32 = lib32.relu()
    scale = float(ref.abs().max())
    err = float((got.double() - ref).abs().max()) / scale
    err_lib = float((lib32.double() - ref).abs().max()) / scale
    r = _elementwise_err(got, x, w, b, z, relu_in, relu_out)
    print(f'[{NB},{Cin}->{Cout},{H}x{W}] {epi}: wgmma 3xTF32 err {err:.2e}, cuDNN fp32 err {err_lib:.2e} (relative to max |y|); '
          f'per element {r / U:.2f} u')
    # fp32 accumulation over K = 9 Cin terms leaves cuDNN's own fp32 result ~1e-5 from float64 at these sizes; 3xTF32 must be
    # of that class (measured 1.4x cuDNN's error) -- a plain 1xTF32 product sits at ~3e-4
    assert err < 4 * err_lib + 2e-6 and err < 6e-5, (err, err_lib)
    assert r <= BAR_TF32, r / U


def test_conv3x3_tc_rejects_unsupported_geometry():
    import cutie_b200.kernels as K_
    assert not K_.conv_tc_eligible(torch.empty(32, 32, 3, 3)) and not K_.conv_tc_eligible(torch.empty(128, 48, 3, 3))
    assert K_.conv_tc_eligible(torch.empty(128, 32, 3, 3)) and not K_.conv_tc_eligible(torch.empty(128, 32, 3, 3), stride=(3, 3))
    img = K_.conv_weight_image(torch.randn(128, 32, 3, 3, device='cuda'))
    with pytest.raises(K_.KernelError):
        K_.conv_tc(torch.randn(1, 33, 4, 4, device='cuda'), img, None, 128)


CASES_1x1 = [
    # NB, Cin, Cout, H, W, stride
    (1, 1024, 256, 30, 54, 1),     # ResNet-50 layer3 bottleneck entry
    (1, 256, 1024, 30, 54, 1),     # ... and exit
    (1, 64, 256, 120, 216, 1),
    (3, 256, 256, 30, 54, 1),      # pixel_init_proj
    (1, 512, 1024, 60, 108, 2),    # layer3 projection shortcut (stride 2)
    (2, 64, 128, 9, 7, 2),         # odd sizes, stride 2
    (1, 32, 64, 3, 5, 1),          # fewer than 16 pixels
]

# (channels-last input, epilogue); the first two keep their original ids
LAYOUT_EPI_1x1 = [pytest.param(False, 'residual+relu_out', id='False'), pytest.param(True, 'residual+relu_out', id='True'),
                  pytest.param(False, 'plain', id='False-plain'), pytest.param(True, 'no_bias+relu_in', id='True-no_bias+relu_in')]


@pytest.mark.parametrize('NB,Cin,Cout,H,W,stride', CASES_1x1)
@pytest.mark.parametrize('cl,epi', LAYOUT_EPI_1x1)
def test_conv1x1_tc_is_fp32_class_accurate(NB, Cin, Cout, H, W, stride, cl, epi):
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device='cuda').manual_seed(Cin + H)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g) * 1.5
    w = torch.randn(Cout, Cin, 1, 1, device='cuda', generator=g) * (2.0 / Cin) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    z = torch.randn(NB, Cout, Ho, Wo, device='cuda', generator=g)
    if 'residual' not in epi:
        z = None
    if 'no_bias' in epi:
        b = None
    relu_in, relu_out = 'relu_in' in epi, 'relu_out' in epi
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    img = K_.conv_weight_image(w)
    got = K_.conv_tc(x, img, b, Cout, ksize=1, stride=stride, residual=z, relu_in=relu_in, relu_out=relu_out)   # z: NCHW
    assert got.shape == (NB, Cout, Ho, Wo)
    assert got.is_contiguous(memory_format=torch.channels_last if cl and Cout > 1 and Ho * Wo > 1 else torch.contiguous_format)
    pre = x.relu() if relu_in else x
    ref = F.conv2d(pre.double(), w.double(), b.double() if b is not None else None, stride=stride)
    lib32 = F.conv2d(pre, w, b, stride=stride)
    if z is not None:
        ref, lib32 = ref + z.double(), lib32 + z
    if relu_out:
        ref, lib32 = ref.relu(), lib32.relu()
    scale = float(ref.abs().max())
    err = float((got.double() - ref).abs().max()) / scale
    err_lib = float((lib32.double() - ref).abs().max()) / scale
    r = _elementwise_err(got, x, w, b, z, relu_in, relu_out, stride)
    print(f'1x1 [{NB},{Cin}->{Cout},{H}x{W}] s{stride} cl={cl} {epi}: wgmma 3xTF32 err {err:.2e}, cuDNN fp32 err {err_lib:.2e}; '
          f'per element {r / U:.2f} u')
    assert err < 4 * err_lib + 2e-6 and err < 6e-5, (err, err_lib)
    assert r <= BAR_TF32, r / U


@pytest.mark.parametrize('NB,Cin,Cout,H,W', [(1, 64, 64, 120, 216), (1, 256, 256, 30, 54), (2, 128, 128, 17, 23)])
def test_conv3x3_tc_channels_last_in_and_out(NB, Cin, Cout, H, W):
    """The trunks run channels-last: same kernel, strided addressing, residual in the other layout."""
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device='cuda').manual_seed(7)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) * (2.0 / (9 * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    z = torch.randn(NB, Cout, H, W, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)
    img = K_.conv_weight_image(w)
    dense = K_.conv_tc(x, img, b, Cout, residual=z, relu_in=True, relu_out=True)
    last = K_.conv_tc(x.contiguous(memory_format=torch.channels_last), img, b, Cout, residual=z.contiguous(), relu_in=True,
                      relu_out=True)
    assert dense.is_contiguous() and last.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(dense, last.contiguous())            # the same arithmetic whatever the memory format
    ref = (F.conv2d(x.double().relu(), w.double(), b.double(), padding=1) + z.double()).relu()
    assert float((dense.double() - ref).abs().max()) < 1e-5 * float(ref.abs().max())
    r = _elementwise_err(dense, x, w, b, z, relu_in=True, relu_out=True)
    print(f'3x3 [{NB},{Cin}->{Cout},{H}x{W}] channels-last: per element {r / U:.2f} u')
    assert r <= BAR_TF32, r / U


@pytest.mark.parametrize('NB,Cin,Cout,H,W,k', [(1, 1024, 256, 30, 54, 1), (1, 256, 256, 30, 54, 3), (1, 128, 128, 60, 108, 3),
                                               (2, 96, 200, 7, 9, 3), (1, 512, 128, 60, 108, 1), (3, 256, 256, 30, 54, 3)])
@pytest.mark.parametrize('q', [1, 2, 3, 5, 7])
def test_shared_tiles_are_deterministic_and_as_accurate(NB, Cin, Cout, H, W, k, q):
    """Layers with fewer output tiles than SMs are spread over the SMs in (tile, input chunk) units, q per CTA: a CTA's share
    may span two tiles, a tile's shares meet in a workspace and the CTA that arrives last adds them in slot order -- the
    result does not depend on arrival order (runs are bit-identical), the counters come back zero, accuracy is that of the
    one-tile-per-CTA kernel, which is itself bit-identical over launches."""
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    if q > Cin // 32:
        pytest.skip('more units per CTA than chunks per tile')
    g = torch.Generator(device='cuda').manual_seed(q + Cin)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * (2.0 / (k * k * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    z = torch.randn(NB, Cout, H, W, device='cuda', generator=g)
    img = K_.conv_weight_image(w)
    cnt = torch.zeros(8192, dtype=torch.int32, device='cuda')
    ref = (F.conv2d(x.double(), w.double(), b.double(), padding=k // 2) + z.double()).relu()
    scale = float(ref.abs().max())
    ones = [K_.conv_tc(x, img, b, Cout, ksize=k, residual=z, relu_out=True, units_per_cta=Cin // 32) for _ in range(3)]
    assert torch.equal(ones[0], ones[1]) and torch.equal(ones[0], ones[2])
    one = ones[0]
    e_one = float((one.double() - ref).abs().max()) / scale
    r_one = _elementwise_err(one, x, w, b, z, relu_out=True)
    assert r_one <= BAR_TF32, r_one / U
    for xx, zz in ((x, z), (x.contiguous(), z), (x, z.contiguous(memory_format=torch.channels_last))):   # staged NCHW / CL / direct
        outs = [K_.conv_tc(xx, img, b, Cout, ksize=k, residual=zz, relu_out=True, units_per_cta=q, counters=cnt) for _ in range(3)]
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
        assert int(cnt.abs().max()) == 0
        e = float((outs[0].double() - ref).abs().max()) / scale
        assert e < 2 * e_one + 1e-6, (e, e_one)
        r = _elementwise_err(outs[0], xx, w, b, zz, relu_out=True)
        assert r <= BAR_TF32, r / U
    print(f'{k}x{k} [{NB},{Cin}->{Cout},{H}x{W}] {q} units per CTA: err {e:.2e} (whole tiles {e_one:.2e}); per element '
          f'{r / U:.2f} u (whole tiles {r_one / U:.2f} u)')


def test_conv_plan_spreads_small_layers_over_the_sms():
    import ctypes
    import cutie_b200.kernels as K_
    plan = (ctypes.c_int64 * 6)()
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def p(NB, Cin, Cout, H, W, k, s=1):
        assert K_.lib().cutie_conv_plan(ctypes.c_int64(NB), ctypes.c_int64(Cin), ctypes.c_int64(Cout), ctypes.c_int64(H),
                                        ctypes.c_int64(W), k, s, 0, plan) == 0
        return tuple(plan)                                       # T, N, C, q, CTAs, workspace floats
    T, N, C, q, ctas, ws = p(3, 256, 256, 30, 54, 3)              # PixelFFN: 90 tiles x 8 chunks
    assert (T, N, C) == (90, 112, 8) and q == 8 and ctas == 90 and ws == 0          # 90 x 2 > SMs: whole tiles
    T, N, C, q, ctas, ws = p(1, 64, 256, 120, 216, 1)             # 406 tiles: one whole tile per CTA, no workspace
    assert q == C == 2 and ctas == T == 406 and ws == 0
    T, N, C, q, ctas, ws = p(1, 1024, 256, 30, 54, 1)
    assert T == 26 and C == 32 and ctas <= sms and q * ctas >= T * C and C % q == 0 and ws > 0


CASES_S2 = [
    # NB, Cin, Cout, H, W (input)
    (1, 128, 128, 120, 216), (1, 256, 256, 60, 108), (3, 64, 128, 120, 216), (3, 128, 256, 60, 108), (2, 32, 64, 9, 7),
    (1, 64, 128, 10, 12), (1, 32, 128, 1, 1),
    (1, 64, 128, 1, 300), (1, 64, 128, 300, 1),        # a single row / column: 1 x 150 and 150 x 1 outputs
]

# (channels-last input, epilogue); the first two keep their original ids
LAYOUT_EPI_S2 = [pytest.param(False, 'relu_out', id='False'), pytest.param(True, 'relu_out', id='True'),
                 pytest.param(True, 'relu_in+residual', id='True-relu_in+residual'),
                 pytest.param(False, 'no_bias', id='False-no_bias')]


@pytest.mark.parametrize('NB,Cin,Cout,H,W', CASES_S2)
@pytest.mark.parametrize('cl,epi', LAYOUT_EPI_S2)
def test_conv3x3_stride2_tc(NB, Cin, Cout, H, W, cl, epi):
    """The trunks' four stride-2 3x3 layers: four parity planes of the input window read through row-shifted descriptors."""
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device='cuda').manual_seed(H + Cin)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g) * 1.5
    w = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) * (2.0 / (9 * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    z = torch.randn(NB, Cout, Ho, Wo, device='cuda', generator=g) if 'residual' in epi else None
    if epi == 'no_bias':
        b = None
    relu_in, relu_out = 'relu_in' in epi, 'relu_out' in epi
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    assert K_.conv_tc_eligible(w, stride=(2, 2))
    img = K_.conv_weight_image(w)
    got = K_.conv_tc(x, img, b, Cout, ksize=3, stride=2, residual=z, relu_in=relu_in, relu_out=relu_out)
    pre = x.relu() if relu_in else x
    ref = F.conv2d(pre.double(), w.double(), b.double() if b is not None else None, stride=2, padding=1)
    lib32 = F.conv2d(pre, w, b, stride=2, padding=1)
    if z is not None:
        ref, lib32 = ref + z.double(), lib32 + z
    if relu_out:
        ref, lib32 = ref.relu(), lib32.relu()
    assert got.shape == ref.shape
    scale = float(ref.abs().max())
    err = float((got.double() - ref).abs().max()) / scale
    err_lib = float((lib32.double() - ref).abs().max()) / scale
    r = _elementwise_err(got, x, w, b, z, relu_in, relu_out, stride=2)
    print(f'3x3 s2 [{NB},{Cin}->{Cout},{H}x{W}] cl={cl} {epi}: wgmma 3xTF32 err {err:.2e}, cuDNN fp32 err {err_lib:.2e}; '
          f'per element {r / U:.2f} u')
    assert err < 4 * err_lib + 2e-6 and err < 6e-5, (err, err_lib)
    assert r <= BAR_TF32, r / U


# Defects a main-loop rewrite can make, emulated through the public API: the lo term of the 3xTF32 split missing for all
# weights, for one tap, for one 32-channel input chunk or for the second MMA warpgroup's output channels (a weight image
# built from tf32_rna(w) on that slice has a zero lo plane there), or for the activations (x pre-rounded to tf32).
MUTANT_LAYERS = [
    # NB, Cin, Cout, H, W, k, stride, units per CTA (None: the plan's)
    (1, 64, 128, 23, 40, 3, 1, None),
    (2, 64, 128, 33, 47, 3, 2, None),
    (1, 64, 256, 30, 54, 1, 1, None),
    (1, 64, 128, 30, 54, 3, 1, 1),          # shared tiles: a tile's two chunks from two CTAs
    (1, 512, 256, 23, 40, 3, 1, None),      # 16 chunks: one chunk is 1/16 of K
    (3, 512, 768, 30, 54, 3, 1, None),      # sensory update
    (1, 1024, 256, 30, 54, 1, 1, None),     # 32 chunks; the plan shares the tiles
]
MUTANTS = ['none', 'w_lo_all', 'w_lo_centre_tap', 'w_lo_chunk1', 'w_lo_co64_127', 'x_tf32']


@pytest.mark.parametrize('NB,Cin,Cout,H,W,k,stride,q', MUTANT_LAYERS)
@pytest.mark.parametrize('mutant', MUTANTS)
def test_per_element_bar_rejects_lo_term_defects(NB, Cin, Cout, H, W, k, stride, q, mutant):
    """The real kernel ('none') passes the per-element bar; each defect scores at least 4x it against the unrounded
    float64 truth.  The norm-wise metric of the tests above, and whether its bar would pass the result, are printed
    beside it: that bar moves with cuDNN's own error on the day."""
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    g = torch.Generator(device='cuda').manual_seed(NB * 1000 + Cin + H + k)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g) * 1.5
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * (2.0 / (k * k * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    c = k // 2
    if mutant == 'w_lo_centre_tap' and k == 1:
        pytest.skip('a 1x1 layer has one tap: the same image as w_lo_all')
    xm, wm = x, w.clone()
    if mutant == 'w_lo_all':
        wm = tf32_rna(w)
    elif mutant == 'w_lo_centre_tap':
        wm[:, :, c, c] = tf32_rna(w[:, :, c, c])
    elif mutant == 'w_lo_chunk1':
        wm[:, 32:64] = tf32_rna(w[:, 32:64])
    elif mutant == 'w_lo_co64_127':
        wm[64:128] = tf32_rna(w[64:128])
    elif mutant == 'x_tf32':
        xm = tf32_rna(x)
    got = K_.conv_tc(xm, K_.conv_weight_image(wm), b, Cout, ksize=k, stride=stride, units_per_cta=q)
    r = _elementwise_err(got, x, w, b, stride=stride)
    ref = F.conv2d(x.double(), w.double(), b.double(), stride=stride, padding=c)
    old = float((got.double() - ref).abs().max()) / float(ref.abs().max())
    old_lib = float((F.conv2d(x, w, b, stride=stride, padding=c).double() - ref).abs().max()) / float(ref.abs().max())
    old_pass = old < 4 * old_lib + 2e-6 and old < 6e-5
    print(f'{k}x{k} s{stride} [{NB},{Cin}->{Cout},{H}x{W}] q={q} {mutant}: per element {r / U:.1f} u '
          f'({r / BAR_TF32:.1f}x the bar); norm-wise {old:.2e} (cuDNN fp32 {old_lib:.2e}: the norm-wise bar would '
          f'{"pass" if old_pass else "reject"} it)')
    if mutant == 'none':
        assert r <= BAR_TF32, r / U
    else:
        assert r >= 4 * BAR_TF32, r / U


def _image_tf32_restated(w: torch.Tensor) -> torch.Tensor:
    """The 3xTF32 operand image in Python: per (128-channel tile, 32-channel chunk, tap) a hi plane and then a lo plane of
    [128 rows x 128 B], row = output channel (zero past Cout), 16-byte piece k4 (channels 4 k4 .. 4 k4 + 3 of the chunk)
    stored at piece k4 ^ (row & 7); hi = tf32_rna(w), lo = tf32_rna(w - hi)."""
    Cout, Cin, k, _ = w.shape
    cots, chunks, taps = (Cout + 127) // 128, Cin // 32, k * k
    wp = torch.zeros(cots * 128, Cin, taps, dtype=torch.float32, device=w.device)
    wp[:Cout] = w.reshape(Cout, Cin, taps)
    hi = tf32_rna(wp)
    planes = torch.stack([hi, tf32_rna(wp - hi)])                                         # [plane, row, Cin, tap]
    blocks = planes.reshape(2, cots, 128, chunks, 8, 4, taps).permute(1, 3, 6, 0, 2, 4, 5)  # [cot, chunk, tap, plane, row, piece, 4]
    out = torch.empty_like(blocks)
    rows = torch.arange(128, device=w.device)
    for piece in range(8):
        out[:, :, :, :, rows, piece ^ (rows & 7)] = blocks[:, :, :, :, rows, piece]
    return out.contiguous().reshape(-1)


# fp32 bit patterns where rounding to tf32 can go wrong: ties (rna rounds them away from zero, ties-to-even would not),
# subnormals, and values at the top of the range (the largest ones round up to inf)
SPECIAL_BITS = [0x3F801000, 0xBF801000, 0x3F803000, 0x3F800FFF, 0x3F801001, 0x00000001, 0x00001000, 0x80001000, 0x00003000,
                0x007FF000, 0x007FFFFF, 0x00800000, 0x7F7FE000, 0x7F7FEFFF, 0x7F7FF000, 0xFF7FF000, 0x7F7FFFFF]


@pytest.mark.parametrize('Cout,Cin,k', [(128, 32, 3), (200, 64, 3), (256, 1024, 1), (64, 96, 1)])
def test_conv_weight_image_layout(Cout, Cin, k):
    import cutie_b200.kernels as K_
    g = torch.Generator(device='cuda').manual_seed(Cout + Cin)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 3
    special = torch.tensor([v - (1 << 32) if v >= 1 << 31 else v for v in SPECIAL_BITS], dtype=torch.int32).view(torch.float32)
    flat = w.view(-1)
    flat[:len(special)] = special.cuda()
    flat[-len(special):] = special.cuda()                     # the last row of the layer
    img = K_.conv_weight_image(w)
    assert img.numel() * 4 == K_.conv_weight_image_bytes(Cout, Cin, k) == (Cout + 127) // 128 * Cin // 32 * k * k * 32768
    got, want = img.view(torch.int32), _image_tf32_restated(w).view(torch.int32)
    bad = (got != want).nonzero().flatten()
    assert bad.numel() == 0, [(int(i), hex(int(got[i]) & 0xFFFFFFFF), hex(int(want[i]) & 0xFFFFFFFF)) for i in bad[:8]]


@pytest.mark.parametrize('f16', [False, True])
def test_conv_tc_bias_must_be_one_float_per_output_channel(f16):
    """A strided bias view is copied to a contiguous tensor before the launch (same bits as passing that copy); a bias of
    the wrong shape or type is refused rather than read out of bounds."""
    import cutie_b200.kernels as K_
    g = torch.Generator(device='cuda').manual_seed(3)
    x = torch.randn(1, 64, 9, 11, device='cuda', generator=g)
    w = torch.randn(128, 64, 3, 3, device='cuda', generator=g) * 0.06
    b2 = torch.randn(256, device='cuda', generator=g)
    img = K_.conv_weight_image_f16(w) if f16 else K_.conv_weight_image(w)
    got = K_.conv_tc(x, img, b2[::2], 128, f16=f16)
    assert torch.equal(got, K_.conv_tc(x, img, b2[::2].contiguous(), 128, f16=f16))
    for bad in (b2[:127], b2[:129], b2[:128].reshape(1, 128), b2[:128].double()):
        with pytest.raises(K_.KernelError):
            K_.conv_tc(x, img, bad, 128, f16=f16)


ODD_LAYOUTS = [
    # what, NB, Cin, Cout, k, stride, units per CTA (None: whole tiles)
    ('x_at_4B', 2, 64, 128, 3, 1, None),
    ('x_at_4B', 2, 64, 128, 3, 2, None),
    ('x_at_4B', 2, 64, 128, 1, 1, None),
    ('cout66', 1, 128, 66, 3, 1, None),
    ('cout66', 1, 128, 66, 3, 1, 2),
    ('cout130', 1, 128, 130, 3, 1, None),
    ('cout130', 1, 128, 130, 3, 1, 3),
    ('bias_at_4B', 1, 128, 128, 3, 1, None),
    ('bias_at_4B', 1, 128, 128, 1, 1, 1),
]


@pytest.mark.parametrize('what,NB,Cin,Cout,k,stride,q', ODD_LAYOUTS)
@pytest.mark.parametrize('f16', [False, True])
def test_conv_tc_channels_last_off_the_vector_paths(what, NB, Cin, Cout, k, stride, q, f16):
    """Channels-last tensors the 16-byte paths cannot take: an input whose data is only 4-byte aligned (the producers read
    it channel by channel), an output with Cout % 4 != 0 or a bias that is not 16-byte aligned (the element-wise
    epilogue, straight from the accumulators or after shared tiles).  The bits are those of the dense NCHW call with an
    aligned bias, and every element is within the per-element bar."""
    import cutie_b200.kernels as K_
    H, W = 17, 23
    g = torch.Generator(device='cuda').manual_seed(Cout + k + stride)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g) * 1.5
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * (2.0 / (k * k * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    z = torch.randn(NB, Cout, Ho, Wo, device='cuda', generator=g)
    img = K_.conv_weight_image_f16(w) if f16 else K_.conv_weight_image(w)
    q = q or Cin // 32

    def conv(xx, bb, zz):
        return K_.conv_tc(xx, img, bb, Cout, ksize=k, stride=stride, residual=zz, relu_out=True, units_per_cta=q, f16=f16)
    dense = conv(x, b, z)
    xl = x.contiguous(memory_format=torch.channels_last)
    bl = b
    if what == 'x_at_4B':
        xl = torch.empty(x.numel() + 1, device='cuda')[1:].view(NB, H, W, Cin).permute(0, 3, 1, 2)
        xl.copy_(x)
        assert xl.is_contiguous(memory_format=torch.channels_last) and xl.data_ptr() % 16 == 4
    if what == 'bias_at_4B':
        bl = torch.empty(Cout + 1, device='cuda')[1:]
        bl.copy_(b)
        assert bl.data_ptr() % 16 == 4
    got = conv(xl, bl, z.contiguous(memory_format=torch.channels_last))
    assert got.is_contiguous(memory_format=torch.channels_last)
    assert torch.equal(got, dense)
    r = _elementwise_err(got, x, w, b, z, relu_out=True, stride=stride, f16=f16)
    print(f'{what} {k}x{k} s{stride} [{NB},{Cin}->{Cout},{H}x{W}] q={q} {"fp16" if f16 else "3xTF32"}: per element {r / U:.2f} u')
    assert r <= (BAR_F16 if f16 else BAR_TF32), r / U
