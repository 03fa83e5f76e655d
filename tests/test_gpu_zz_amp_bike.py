"""InferenceCore.step under CUDA autocast, as the reference's own drivers call it (scripting_demo.py:12-13 decorates its
whole loop with @torch.cuda.amp.autocast(); the GUI and eval_vos.py open autocast when `amp: True`).  The step runs
with autocast off and the optimised model's tensor-core convolutions in their FP16-operand form ('tc16').

Named to sort after the other bike test and before test_gpu_zzz_conv_timing.py (cuDNN autotuner persistence)."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN
from tests.test_gpu_zz_cfg1_bike import _inputs, _like_a_fresh_process, _net, _per_frame, _reference_on_this_gpu

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900, method='thread')]


def _fp32_settings():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = False


def _optimised():
    cfg, net = _net()
    return cfg, net.cuda().optimize_for_inference()


def _demo(cfg, net, frames, mask, objects, graphs, amp=True):
    """scripting_demo.py:12-58 -- its two decorators verbatim -- on the given frames; returns (outputs, logits of the
    propagated frames, output masks), all on the CPU."""
    from cutie_b200.inference.inference_core import InferenceCore
    outs, logits, masks = [], [], []

    @torch.inference_mode()
    @torch.cuda.amp.autocast(enabled=amp)
    def main():
        processor = InferenceCore(net, cfg=cfg, use_cuda_graphs=graphs)
        processor.max_internal_size = 480
        m = mask.cuda()
        for ti, frame in enumerate(frames):
            image = frame.cuda().float()
            if ti == 0:
                output_prob = processor.step(image, m, objects=objects)
            else:
                output_prob = processor.step(image)
                logits.append(processor.last_logits.clone().cpu())
            m = processor.output_prob_to_mask(output_prob)
            outs.append(output_prob.cpu())
            masks.append(m.cpu())
    main()
    return outs, logits, masks


@pytest.mark.parametrize('graphs', [False, True])
def test_scripting_demo_loop_runs_under_autocast(graphs):
    _fp32_settings()
    g = np.load(os.path.join(GOLDEN, 'cfg1_bike.npz'))
    frames, mask, objects = _inputs(g)
    cfg, net = _optimised()
    outs, logits, _ = _demo(cfg, net, frames, mask, objects, graphs)
    for o in outs:
        assert o.dtype == torch.float32 and tuple(o.shape) == (3, 480, 854) and torch.isfinite(o).all()
    assert all(torch.isfinite(x).all() for x in logits)
    rep = net.conv_epilogues.report()['layers']
    print(f'graphs={graphs}: forms {rep}')
    assert rep.get('tc16', 0) > 0 and rep.get('tc', 0) > 0     # the two sensory transforms keep the fp32-class form


_REF_AMP = {}


def _reference_under_autocast(frames, mask, objects):
    """The UNMODIFIED reference with every step inside torch.autocast('cuda', dtype=torch.float16), on this GPU."""
    if 'amp' not in _REF_AMP:
        _reference_on_this_gpu(frames, mask, objects, exact_similarity=True)     # fails / skips without a reference
        from tests.ref_runner_amp import run_reference_clip_amp
        _REF_AMP['amp'] = run_reference_clip_amp(frames, mask, objects, device='cuda', max_internal_size=480)
    return _REF_AMP['amp']


def test_amp_first_propagated_frame_is_as_close_as_the_reference_under_autocast():
    """Against the float64-similarity fp32 reference on this GPU: the first propagated frame of our amp step is at least as
    close as the unmodified reference's own autocast run; mask pixels differing on frames 0-1 are no more than
    max(2e-4, the reference-under-autocast's fraction).  Later frames and amp vs fp32 are reported."""
    _fp32_settings()
    _like_a_fresh_process()
    g = np.load(os.path.join(GOLDEN, 'cfg1_bike.npz'))
    frames, mask, objects = _inputs(g)
    exact = _reference_on_this_gpu(frames, mask, objects, exact_similarity=True)
    ref_amp = _reference_under_autocast(frames, mask, objects)
    cfg, net = _optimised()
    _, ours, ours_masks = _demo(cfg, net, frames, mask, objects, graphs=False)
    _, ours32, _ = _demo(cfg, net, frames, mask, objects, graphs=False, amp=False)
    err_ours = _per_frame(ours, exact['logits'][1:])
    err_ref = _per_frame(ref_amp['logits'][1:], exact['logits'][1:])
    err_ours32 = _per_frame(ours32, exact['logits'][1:])
    print(f'max |logit diff| per propagated frame vs the float64-similarity fp32 reference: ours under autocast {err_ours}; '
          f'reference under autocast {err_ref}; ours fp32 {err_ours32}; ours amp vs ours fp32 {_per_frame(ours, ours32)}')
    assert err_ours[0] <= err_ref[0], (err_ours, err_ref)
    for ti in (0, 1):
        ours_d = float((ours_masks[ti] != exact['masks'][ti]).float().mean())
        ref_d = float((ref_amp['masks'][ti] != exact['masks'][ti]).float().mean())
        print(f'frame {ti}: mask pixels differing, ours amp {ours_d:.2e}, reference amp {ref_d:.2e}')
        assert ours_d <= max(2e-4, ref_d), (ti, ours_d, ref_d)


def _e2e_net(cfg):
    from cutie_b200.model.cutie import CUTIE
    from oracle.synth import synthetic_state_dict
    net = CUTIE(cfg).eval()
    net.load_state_dict(synthetic_state_dict(net.state_dict(), 0))
    return net.cuda().optimize_for_inference()


def test_amp_graph_path_matches_eager():
    """Under autocast, graph replays equal the eager amp path (same kernels, same order) and account for the same number
    of cutie_b200 kernels, as the fp32 graph path does."""
    from cutie_b200.config import default_config
    from cutie_b200.inference.inference_core import InferenceCore
    import cutie_b200.kernels as K_
    from oracle.synth import synthetic_video
    _fp32_settings()
    cfg = default_config(mem_every=3, max_mem_frames=3)
    net = _e2e_net(cfg)
    eager, graphed = InferenceCore(net, cfg=cfg), InferenceCore(net, cfg=cfg, use_cuda_graphs=True)
    frames, mask = synthetic_video(9, 240, 432, 3, seed=7)
    with torch.inference_mode(), torch.autocast('cuda', dtype=torch.float16):
        for ti in range(9):
            a = frames[ti].cuda()
            if ti == 0:
                pe = eager.step(a, mask.cuda(), objects=[1, 2, 3])
                pg = graphed.step(a, mask.cuda(), objects=[1, 2, 3])
            else:
                n0 = K_.LAUNCH_COUNT
                pe = eager.step(a)
                n_eager = K_.LAUNCH_COUNT - n0
                ncap = len(graphed._graphs._seg) + len(graphed._graphs._enc)
                pg = graphed.step(a)
                n_graph = K_.LAUNCH_COUNT - n0 - n_eager
                if len(graphed._graphs._seg) + len(graphed._graphs._enc) == ncap:
                    assert n_graph == n_eager
                assert float((eager.last_logits - graphed.last_logits).abs().max()) < 2e-4
            assert pe.dtype == pg.dtype == torch.float32
            assert float((pe - pg).abs().max()) < 1e-4
    assert all(k[-1] for k in graphed._graphs._seg) and all(k[-1] for k in graphed._graphs._enc)    # amp captures only
    assert net.conv_epilogues.report()['layers'].get('tc16', 0) > 0


def test_switching_autocast_between_steps_graphed_matches_eager():
    """A graphed processor (with encoder look-ahead) whose caller turns autocast on and off between steps gives what an
    eager processor given the same switches gives: fp32 and amp captures are never mixed up, and a look-ahead encoded in
    the other mode is not used."""
    from cutie_b200.config import default_config
    from cutie_b200.inference.inference_core import InferenceCore
    from oracle.synth import synthetic_video
    _fp32_settings()
    cfg = default_config(mem_every=3, max_mem_frames=3)
    net = _e2e_net(cfg)
    eager, graphed = InferenceCore(net, cfg=cfg), InferenceCore(net, cfg=cfg, use_cuda_graphs=True)
    T = 10
    frames, mask = synthetic_video(T + 1, 240, 432, 3, seed=9)
    cf = [f.cuda() for f in frames]
    amp_at = [False, True, True, False, True, False, False, True, True, False]
    with torch.inference_mode():
        for ti in range(T):
            with torch.autocast('cuda', dtype=torch.float16, enabled=amp_at[ti]):
                if ti == 0:
                    pe = eager.step(cf[0], mask.cuda(), objects=[1, 2, 3])
                    pg = graphed.step(cf[0], mask.cuda(), objects=[1, 2, 3], next_image=cf[1])
                else:
                    pe = eager.step(cf[ti])
                    pg = graphed.step(cf[ti], next_image=cf[ti + 1])
                    assert float((eager.last_logits - graphed.last_logits).abs().max()) < 2e-4, ti
            assert float((pe - pg).abs().max()) < 1e-4, ti
    modes = {k[-1] for k in graphed._graphs._seg}
    assert modes == {False, True}, modes
