"""cutie_conv_tc_f16 (csrc/conv_tc.cu, F16 = true): the convolution with FP16 operands and fp32 accumulation that the
model runs under fp16 autocast.  Three bars per geometry:

  * operand rounding is the ONLY error: against float64 conv2d of the fp16-rounded operands (bias and residual exact) it
    must be of the class of cuDNN's fp32 result on the same rounded operands -- the bar of tests/test_gpu_conv_tc.py;
  * per element, against the same rounded-operand truth, its error is within BAR_F16 of the sum of the magnitudes of the
    terms (tests/test_gpu_conv_tc.py, _elementwise_err);
  * it is at least as good as what autocast would have run: against float64 of the ORIGINAL operands its error is within
    1.0x that of cuDNN's fp16 convolution F.conv2d(pre(x).half(), w.half(), b.half())."""
import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_conv_tc import BAR_F16, CASES, CASES_1x1, CASES_S2, LAYOUT_EPI_1x1, LAYOUT_EPI_S2, U, _elementwise_err

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600, method='thread')]

AMP_MARGIN = 1.0                 # measured on an H100: at most 0.94x, typically 0.4x, cuDNN fp16's error


def _epilogue(y, z, relu_out):
    if z is not None:
        y = y + z
    return y.relu() if relu_out else y


def _check(got, x, w, b, z, relu_in, relu_out, stride, what, vs_autocast=True):
    """All three bars (vs_autocast=False: the comparison with autocast is printed, not asserted); returns (error vs the
    rounded-operand truth, error vs the original-operand truth)."""
    pad = w.shape[-1] // 2
    pre = x.relu() if relu_in else x
    xh, wh = pre.half().float(), w.half().float()
    zd = z.double() if z is not None else None
    bd, bh = (b.double(), b.half()) if b is not None else (None, None)
    ref16 = _epilogue(F.conv2d(xh.double(), wh.double(), bd, stride=stride, padding=pad), zd, relu_out)
    lib32 = _epilogue(F.conv2d(xh, wh, b, stride=stride, padding=pad), z, relu_out)
    ref = _epilogue(F.conv2d(pre.double(), w.double(), bd, stride=stride, padding=pad), zd, relu_out)
    amp = _epilogue(F.conv2d(pre.half(), w.half(), bh, stride=stride, padding=pad).float(), z, relu_out)
    assert got.shape == ref.shape and got.dtype == torch.float32
    s16, s = float(ref16.abs().max()), float(ref.abs().max())
    err = float((got.double() - ref16).abs().max()) / s16
    err_lib = float((lib32.double() - ref16).abs().max()) / s16
    err_o = float((got.double() - ref).abs().max()) / s
    err_amp = float((amp.double() - ref).abs().max()) / s
    r = _elementwise_err(got, x, w, b, z, relu_in, relu_out, stride, f16=True)
    print(f'{what}: vs rounded operands {err:.2e} (cuDNN fp32 {err_lib:.2e}); vs original operands {err_o:.2e} '
          f'(cuDNN fp16 {err_amp:.2e}, ratio {err_o / err_amp:.2f}); per element vs rounded operands {r / U:.2f} u')
    assert err < 4 * err_lib + 2e-6 and err < 6e-5, (err, err_lib)
    assert err_o <= AMP_MARGIN * err_amp or not vs_autocast, (err_o, err_amp)
    assert r <= BAR_F16, r / U
    return err, err_o


@pytest.mark.parametrize('NB,Cin,Cout,H,W', CASES)
@pytest.mark.parametrize('epi', ['plain', 'relu_in+residual', 'relu_out', 'no_bias'])
def test_conv3x3_tc_f16_error_is_operand_rounding_only(NB, Cin, Cout, H, W, epi):
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
    img = K_.conv_weight_image_f16(w)
    got = K_.conv_tc_f16(x, img, b, Cout, residual=z, relu_in=relu_in, relu_out=relu_out)
    # Without a bias, the kernel and autocast start from the same fp16 operands (the kernel's edge over autocast is mostly
    # its exact fp32 bias).  On a single output pixel, 128 values, which of the two has the larger maximum error is then
    # chance: measured 1.05x at 64 -> 128, with the kernel 0.7 U from the rounded-operand truth.
    vs_autocast = b is not None or H * W > 1
    _check(got, x, w, b, z, relu_in, relu_out, 1, f'3x3 [{NB},{Cin}->{Cout},{H}x{W}] {epi}', vs_autocast)


@pytest.mark.parametrize('NB,Cin,Cout,H,W,stride', CASES_1x1)
@pytest.mark.parametrize('cl,epi', LAYOUT_EPI_1x1)
def test_conv1x1_tc_f16(NB, Cin, Cout, H, W, stride, cl, epi):
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
    got = K_.conv_tc_f16(x, K_.conv_weight_image_f16(w), b, Cout, ksize=1, stride=stride, residual=z, relu_in=relu_in,
                         relu_out=relu_out)
    assert got.is_contiguous(memory_format=torch.channels_last if cl and Cout > 1 and Ho * Wo > 1 else torch.contiguous_format)
    _check(got, x, w, b, z, relu_in, relu_out, stride, f'1x1 [{NB},{Cin}->{Cout},{H}x{W}] s{stride} cl={cl} {epi}')


@pytest.mark.parametrize('NB,Cin,Cout,H,W', CASES_S2)
@pytest.mark.parametrize('cl,epi', LAYOUT_EPI_S2)
def test_conv3x3_stride2_tc_f16(NB, Cin, Cout, H, W, cl, epi):
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
    got = K_.conv_tc_f16(x, K_.conv_weight_image_f16(w), b, Cout, ksize=3, stride=2, residual=z, relu_in=relu_in,
                         relu_out=relu_out)
    _check(got, x, w, b, z, relu_in, relu_out, 2, f'3x3 s2 [{NB},{Cin}->{Cout},{H}x{W}] cl={cl} {epi}')


@pytest.mark.parametrize('NB,Cin,Cout,H,W,k', [(1, 1024, 256, 30, 54, 1), (1, 256, 256, 30, 54, 3), (2, 96, 200, 7, 9, 3),
                                               (3, 256, 256, 30, 54, 3)])
@pytest.mark.parametrize('q', [1, 2, 3, 5])
def test_conv_tc_f16_shared_tiles_are_repeatable(NB, Cin, Cout, H, W, k, q):
    """(tile, input chunk) shares meeting in the workspace: bit-identical over three launches, counters back to zero,
    accuracy that of whole tiles, which are bit-identical over launches too."""
    import cutie_b200.kernels as K_
    torch.backends.cudnn.allow_tf32 = False
    if q > Cin // 32:
        pytest.skip('more units per CTA than chunks per tile')
    g = torch.Generator(device='cuda').manual_seed(q + Cin)
    x = torch.randn(NB, Cin, H, W, device='cuda', generator=g).contiguous(memory_format=torch.channels_last)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * (2.0 / (k * k * Cin)) ** 0.5
    b = torch.randn(Cout, device='cuda', generator=g)
    z = torch.randn(NB, Cout, H, W, device='cuda', generator=g)
    img = K_.conv_weight_image_f16(w)
    cnt = torch.zeros(8192, dtype=torch.int32, device='cuda')
    ones = [K_.conv_tc_f16(x, img, b, Cout, ksize=k, residual=z, relu_out=True, units_per_cta=Cin // 32) for _ in range(3)]
    assert torch.equal(ones[0], ones[1]) and torch.equal(ones[0], ones[2])
    one = ones[0]
    e_one, _ = _check(one, x, w, b, z, False, True, 1, f'{k}x{k} [{NB},{Cin}->{Cout},{H}x{W}] whole tiles')
    for xx, zz in ((x, z), (x.contiguous(), z), (x, z.contiguous(memory_format=torch.channels_last))):
        outs = [K_.conv_tc_f16(xx, img, b, Cout, ksize=k, residual=zz, relu_out=True, units_per_cta=q, counters=cnt)
                for _ in range(3)]
        assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])
        assert int(cnt.abs().max()) == 0
        e, _ = _check(outs[0], xx, w, b, zz, False, True, 1, f'{k}x{k} [{NB},{Cin}->{Cout},{H}x{W}] {q} units per CTA')
        assert e < 2 * e_one + 1e-6, (e, e_one)


def _image_f16_restated(w: torch.Tensor) -> torch.Tensor:
    """The fp16 operand image in Python: per (128-channel tile, 32-channel chunk, tap) a [128 rows x 64 B] block, row =
    output channel, 16-byte piece p (channels 8p .. 8p + 7 of the chunk) stored at piece p ^ ((row >> 1) & 3)."""
    Cout, Cin, k, _ = w.shape
    cots, chunks, taps = (Cout + 127) // 128, Cin // 32, k * k
    wp = torch.zeros(cots * 128, Cin, taps, dtype=torch.float16, device=w.device)
    wp[:Cout] = w.reshape(Cout, Cin, taps).half()
    blocks = wp.reshape(cots, 128, chunks, 4, 8, taps).permute(0, 2, 5, 1, 3, 4)      # [cot, chunk, tap, row, piece, 8]
    out = torch.empty_like(blocks)
    rows = torch.arange(128, device=w.device)
    for piece in range(4):
        out[:, :, :, rows, piece ^ ((rows >> 1) & 3)] = blocks[:, :, :, rows, piece]
    return out.contiguous().view(torch.uint8).reshape(-1)


@pytest.mark.parametrize('Cout,Cin,k', [(128, 32, 3), (200, 64, 3), (256, 1024, 1), (64, 96, 1)])
def test_conv_weight_image_f16_layout(Cout, Cin, k):
    import cutie_b200.kernels as K_
    g = torch.Generator(device='cuda').manual_seed(Cout + Cin)
    w = torch.randn(Cout, Cin, k, k, device='cuda', generator=g) * 3
    w[0, 0, 0, 0] = 1e6                                      # overflows fp16: inf, as Tensor.half() gives
    img = K_.conv_weight_image_f16(w)
    assert img.numel() * 4 == K_.conv_weight_image_bytes(Cout, Cin, k, f16=True) == (Cout + 127) // 128 * Cin // 32 * k * k * 8192
    assert torch.equal(img.view(torch.uint8), _image_f16_restated(w))


def test_conv_tc_f16_rejects_unsupported_geometry_and_foreign_images():
    import cutie_b200.kernels as K_
    w = torch.randn(128, 32, 3, 3, device='cuda')
    img16 = K_.conv_weight_image_f16(w)
    with pytest.raises(K_.KernelError):
        K_.conv_tc_f16(torch.randn(1, 33, 4, 4, device='cuda'), img16, None, 128)
    with pytest.raises(K_.KernelError):                      # a 3xTF32 image is not an fp16 one, and the reverse
        K_.conv_tc_f16(torch.randn(1, 32, 4, 4, device='cuda'), K_.conv_weight_image(w), None, 128)
    with pytest.raises(K_.KernelError):
        K_.conv_tc(torch.randn(1, 32, 4, 4, device='cuda'), img16, None, 128)
    with pytest.raises(K_.KernelError):                      # 1x1 image for a 3x3 call
        K_.conv_tc_f16(torch.randn(1, 32, 4, 4, device='cuda'), K_.conv_weight_image_f16(w[:, :, :1, :1]), None, 128)
