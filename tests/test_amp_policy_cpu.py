"""The mixed-precision policy of InferenceCore.step, driven on the CPU: the autocast reader is substituted (without a GPU
torch.autocast('cuda') disables itself), the device forms of the convolution fuser are emulated ('tc16' = the 'tc'
emulation on fp16-rounded operands), graphs are stand-ins (tests/test_graph_path_cpu.py).  What is tested is the wiring:
which layers take which form in which mode, that nothing else changes, graph keys and the look-ahead per mode, and the
host-side validation of the new C-ABI entry points."""
import ctypes

import pytest
import torch

from cutie_b200.model import fuse
from cutie_b200.model.blocks import DeepSensoryUpdater, MultiScaleSensoryUpdater, ObjResBlock


class _AmpFuser(fuse.ConvEpilogueFuser):
    """Device forms on CPU tensors: 'cudnn' emulated, 'tc' / 'tc16' and 'kernel' through the installed CPU kernels."""

    def _eligible(self, conv, x):
        return self.enabled and conv.bias is not None and x.dim() == 4 and not torch.is_grad_enabled()

    def fused(self, conv, x, z=None):
        y = torch.nn.functional.conv2d(x, conv.weight, conv.bias, conv.stride, conv.padding, conv.dilation, conv.groups)
        return torch.relu(y if z is None else y + z)


@pytest.fixture
def amp_kernels(cpu_kernels, monkeypatch):
    """cpu_kernels plus emulations of the FP16-operand convolution (counted)."""
    import cutie_b200.kernels as K_
    calls = {'tc16': 0}

    def conv_weight_image_f16(weight):
        return weight.detach().half().float()

    def conv_tc_f16(x, weight_image, bias, cout, ksize=3, stride=1, residual=None, relu_in=False, relu_out=False,
                    units_per_cta=None, counters=None):
        calls['tc16'] += 1
        pre = torch.relu(x) if relu_in else x
        return cpu_kernels.conv_tc(pre.half().float(), weight_image, bias, cout, ksize, stride, residual, False, relu_out)
    monkeypatch.setattr(K_, 'conv_weight_image_f16', conv_weight_image_f16)
    monkeypatch.setattr(K_, 'conv_tc_f16', conv_tc_f16)
    return calls


def _blocks():
    torch.manual_seed(3)
    res = ObjResBlock(32, 128).eval()                         # conv1, conv2, 1x1 shortcut: all tensor-core eligible
    ms = MultiScaleSensoryUpdater([32, 32, 32], 32, 32).eval()    # 1x1 32 -> 32 (too narrow: 'kernel'), transform 64 -> 96
    deep = DeepSensoryUpdater(32, 32).eval()                  # transform 64 -> 96
    return res, ms, deep


def _run(res, ms, deep):
    g = torch.randn(1, 2, 32, 4, 6, generator=torch.Generator().manual_seed(1))
    h = torch.randn(1, 2, 32, 4, 6, generator=torch.Generator().manual_seed(2))
    with torch.inference_mode():
        return (res(g), ms(g, torch.nn.functional.interpolate(g[0], scale_factor=2).unsqueeze(0),
                           torch.nn.functional.interpolate(g[0], scale_factor=4).unsqueeze(0), h), deep(g, h))


def test_amp_mode_routes_eligible_layers_to_tc16_and_keeps_the_sensory_transforms(amp_kernels):
    res, ms, deep = _blocks()
    ref = _run(res, ms, deep)
    off, on = _AmpFuser(), _AmpFuser()
    for m in (res, ms, deep):
        fuse.attach_epilogue_fuser(m, off)
    out_off = _run(res, ms, deep)
    for m in (res, ms, deep):
        fuse.attach_epilogue_fuser(m, on)
    with on.amp_mode():
        assert on.amp
        out_on = _run(res, ms, deep)
    assert not on.amp                                          # the mode ends with the block
    # amp off: today's forms; amp on: the eligible layers move to 'tc16', the two transforms and the narrow 1x1s stay
    assert off.report()['layers'] == {'tc': 5, 'kernel': 3}
    assert on.report()['layers'] == {'tc16': 3, 'tc': 2, 'kernel': 3}
    assert amp_kernels['tc16'] == 3
    assert set(on._images16) == {id(res.conv1), id(res.conv2), id(res.downsample)}
    assert set(on._images) == {id(ms.transform), id(deep.transform)}
    for a, b in zip(out_off, ref):
        assert torch.allclose(a, b, atol=1e-5)
    assert torch.allclose(out_on[1], out_off[1], atol=1e-6) and torch.allclose(out_on[2], out_off[2], atol=1e-6)
    assert not torch.allclose(out_on[0], out_off[0], atol=1e-6)                 # fp16 operands: not the fp32 result
    assert torch.allclose(out_on[0], out_off[0], atol=2e-2)


def test_marks_leave_state_dict_unchanged():
    ms, deep = MultiScaleSensoryUpdater([32, 32, 32], 32, 32), DeepSensoryUpdater(32, 32)
    assert ms.transform.amp_fp32 and deep.transform.amp_fp32
    assert set(deep.state_dict()) == {'transform.weight', 'transform.bias'}
    assert not any('amp' in k for k in ms.state_dict())


def _net(cfg, optimise=True):
    from cutie_b200.model.cutie import CUTIE
    from oracle.synth import synthetic_state_dict
    n = CUTIE(cfg).eval()
    n.load_state_dict(synthetic_state_dict(n.state_dict(), 0))
    if not optimise:
        return n
    n = n.optimize_for_inference()
    f = _AmpFuser()
    fuse.attach_epilogue_fuser(n, f)
    object.__setattr__(n, 'conv_epilogues', f)                # the fuser InferenceCore.step switches
    return n


def _autocast_reader(monkeypatch, state):
    import cutie_b200.inference.inference_core as ic
    monkeypatch.setattr(ic, '_autocast_state', lambda: tuple(state))
    return ic


def test_step_policy_per_autocast_state(amp_kernels, monkeypatch):
    from cutie_b200.config import default_config
    from oracle.synth import synthetic_video
    state = [False, torch.float16]
    ic = _autocast_reader(monkeypatch, state)
    cfg = default_config(mem_every=2, max_mem_frames=3)
    net = _net(cfg)
    frames, mask = synthetic_video(4, 96, 160, 2, seed=5)
    seen = []
    orig = net.conv_epilogues.run

    def spy(form, *a, **kw):
        seen.append((form, net.conv_epilogues.amp, torch.is_autocast_enabled('cuda')))
        return orig(form, *a, **kw)
    net.conv_epilogues.run = spy
    fp32 = ic.InferenceCore(net, cfg=cfg)
    amp = ic.InferenceCore(net, cfg=cfg)
    with torch.inference_mode():
        for ti in range(4):
            args, kw = ((frames[0], mask), dict(objects=[1, 2])) if ti == 0 else ((frames[ti],), {})
            state[0] = False
            seen.clear()
            p32 = fp32.step(*args, **kw)
            assert seen and all(f != 'tc16' and not m for f, m, _ in seen)         # no autocast: exactly today's path
            state[0] = True
            seen.clear()
            p16 = amp.step(*args, **kw)
            assert any(f == 'tc16' for f, _, _ in seen) and all(m and not a for _, m, a in seen)
            assert not net.conv_epilogues.amp
            assert p16.dtype == torch.float32 and p16.shape == p32.shape and torch.isfinite(p16).all()
    rep = net.conv_epilogues.report()['layers']
    assert rep['tc16'] > 0 and rep['tc'] > rep['tc16']        # every fp32 triple plus the amp-exempt transforms
    state[1] = torch.bfloat16
    with pytest.raises(NotImplementedError, match='float16'):
        with torch.inference_mode():
            amp.step(frames[1])


def test_unoptimised_model_under_autocast_is_the_fp32_path(cpu_kernels, monkeypatch):
    from cutie_b200.config import default_config
    from oracle.synth import synthetic_video
    state = [False, torch.float16]
    ic = _autocast_reader(monkeypatch, state)
    cfg = default_config(mem_every=2, max_mem_frames=3)
    net = _net(cfg, optimise=False)
    a, b = ic.InferenceCore(net, cfg=cfg), ic.InferenceCore(net, cfg=cfg)
    frames, mask = synthetic_video(3, 96, 160, 2, seed=8)
    with torch.inference_mode():
        for ti in range(3):
            args, kw = ((frames[0], mask), dict(objects=[1, 2])) if ti == 0 else ((frames[ti],), {})
            state[0] = False
            pa = a.step(*args, **kw)
            state[0] = True
            pb = b.step(*args, **kw)
            assert torch.equal(pa, pb)


def test_graph_keys_and_lookahead_follow_the_mode(amp_kernels, monkeypatch):
    """Stand-in graphs: a processor switching autocast between steps (with look-ahead announcements) matches an eager one
    doing the same switches; captures exist per mode."""
    from tests.test_graph_path_cpu import _FakeCaptured, _NoStreams
    import cutie_b200.inference.frame_graphs as fg
    from cutie_b200.config import default_config
    from oracle.synth import synthetic_video
    state = [False, torch.float16]
    ic = _autocast_reader(monkeypatch, state)
    monkeypatch.setattr(fg, '_Captured', _FakeCaptured)
    monkeypatch.setattr(ic, '_graphable', lambda t: True)
    monkeypatch.setattr(ic, '_CudaStreamOps', _NoStreams)
    cfg = default_config(mem_every=3, max_mem_frames=3)
    net = _net(cfg)
    eager, graphed = ic.InferenceCore(net, cfg=cfg), ic.InferenceCore(net, cfg=cfg, use_cuda_graphs=True)
    T = 8
    frames, mask = synthetic_video(T + 1, 96, 160, 2, seed=4)
    amp_at = [False, True, False, True, True, False, False, True]          # memory frames 0, 3, 6: both modes
    with torch.inference_mode():
        for ti in range(T):
            state[0] = amp_at[ti]
            kw = dict(objects=[1, 2]) if ti == 0 else {}
            args = (frames[ti], mask) if ti == 0 else (frames[ti],)
            pe = eager.step(*args, **kw)
            pg = graphed.step(*args, next_image=frames[ti + 1], **kw)
            assert torch.allclose(pg, pe, atol=1e-6), ti
            if ti > 0:
                assert torch.allclose(graphed.last_logits, eager.last_logits, atol=1e-5), ti
    g = graphed._graphs
    for caps in (g._enc, g._seg, g._msk):
        assert {k[-1] for k in caps} == {False, True}


def test_lookahead_announced_in_one_mode_misses_in_the_other():
    from cutie_b200.inference.inference_core import EncoderLookahead
    from tests.test_graph_path_cpu import _NoStreams
    log = []

    def encode(image, slot):
        log.append(slot)
        return ('features', slot)
    la = EncoderLookahead(encode, ops=_NoStreams())
    a, b, c = torch.zeros(3, 2, 2), torch.ones(3, 2, 2), torch.ones(3, 2, 2) * 2
    la.current(0, a.unsqueeze(0), a, mode=False)
    la.ahead(0, b, lambda t: t.unsqueeze(0), mode=True)
    out, hit = la.current(1, b.unsqueeze(0), b, mode=False)           # announced under amp, consumed in fp32: miss
    assert not hit and log[-1] == la.slot == 0
    la.ahead(1, c, lambda t: t.unsqueeze(0), mode=False)
    out, hit = la.current(2, c.unsqueeze(0), c, mode=False)           # same mode: hit, no re-encode
    assert hit and out == ('features', 1) and len(log) == 4


def test_new_entry_points_are_exported_and_validate_on_the_host():
    import __graft_entry__ as ge
    from cutie_b200 import kernels
    ge.build()
    lib = kernels.lib()
    i64 = ctypes.c_int64
    assert lib.cutie_conv_weight_image_f16_bytes(i64(200), i64(64), 3) == 2 * 2 * 9 * 8192
    assert 4 * lib.cutie_conv_weight_image_f16_bytes(i64(256), i64(1024), 1) == lib.cutie_conv_weight_image_bytes(i64(256), i64(1024), 1)
    assert lib.cutie_conv_weight_image_f16_bytes(i64(128), i64(33), 3) == -1
    assert lib.cutie_conv_weight_image_f16_bytes(i64(128), i64(32), 5) == -1
    assert lib.cutie_conv_weight_image_f16(None, i64(128), i64(32), 3, None, None) == -1
    assert b'cutie_conv_weight_image_f16' in lib.cutie_b200_last_error()
    one = ctypes.c_void_p(0x1000)                                       # never dereferenced: validation fails first
    strides = (ctypes.c_int64 * 3)(32 * 16, 16, 1)

    def call(x=one, img=one, y=one, NB=1, Cin=32, k=3, stride=1, ws=None, q=0):
        return lib.cutie_conv_tc_f16(x, strides, img, None, None, None, i64(NB), i64(Cin), i64(128), i64(4), i64(4), k,
                                     stride, 0, 0, y, strides, q, ws, None, None)
    assert call(x=None) == -1 and b'cutie_conv_tc_f16' in lib.cutie_b200_last_error()
    assert call(img=None) == -1
    assert call(Cin=48) == -1 and b'multiple of 32' in lib.cutie_b200_last_error()
    assert call(k=5) == -1 and call(stride=3) == -1 and call(NB=0) == -1
    assert call(Cin=64, q=1) == -1 and b'workspace' in lib.cutie_b200_last_error()   # shared tiles without a workspace
    assert lib.cutie_conv_tc(None, strides, one, None, None, None, i64(1), i64(32), i64(128), i64(4), i64(4), 3, 1, 0, 0,
                             one, strides, 0, None, None, None) == -1
    assert b'cutie_conv_tc:' in lib.cutie_b200_last_error()             # the fp32 entry point still names itself
