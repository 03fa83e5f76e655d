"""fp32 vs fp16-autocast InferenceCore.step on bench.py's cfg 2 stream, one JSON line on stdout.

    python scripts/amp_bench.py [--steps K] [--warmup W] [--blocks B] [--iters I]

* hardware: the card's name and power limit (read-only nvidia-smi query), beside every number;
* step rate: the stream bench.py times (480p, 3 objects, 413 k-token working memory, the same seeds, optimised model,
  CUDA graphs), timed with CUDA events in alternating blocks of K steps -- fp32, then under
  torch.autocast('cuda', dtype=torch.float16), B blocks each -- frames/s per mode;
* conv_tc kernel time per step in each mode: one eager block per mode with every C-ABI call bracketed by CUDA events;
* layer times: cutie_conv_tc (3xTF32), cutie_conv_tc_f16 and cuDNN's fp16 convolution (what autocast runs in the
  reference) on the layers of bench.conv_roofline_bench, CUDA events over I back-to-back launches;
* parity: bench.parity_check (the CPU oracle re-computes one frame from the live state) of an amp step.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import bench  # noqa: E402  (points fd 1 at stderr; bench.emit writes the JSON line to the real stdout)

log = bench.log

# bench.conv_roofline_bench's layers: (name, NB, Cin, Cout, H, W, k, channels-last)
LAYERS = [('PixelFFN / fuser 3x3 256->256 @30x54 x3 objects', 3, 256, 256, 30, 54, 3, False),
          ('sensory update 3x3 512->768 @30x54 x3', 3, 512, 768, 30, 54, 3, False),
          ('decoder 3x3 128->128 @120x216 x3', 3, 128, 128, 120, 216, 3, False),
          ('ResNet-50 layer3 3x3 256->256 @30x54 (channels-last, shared tiles)', 1, 256, 256, 30, 54, 3, True),
          ('ResNet-50 layer3 1x1 1024->256 @30x54 (channels-last, shared tiles)', 1, 1024, 256, 30, 54, 1, True),
          ('ResNet-50 layer1 1x1 64->256 @120x216 + residual (channels-last)', 1, 64, 256, 120, 216, 1, True)]


def hardware():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines() or [','])[0].split(',')[:2]
    return {'name': name.strip(), 'power_limit': power.strip()}


def _timed(fn, iters):
    for _ in range(4):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3


def layer_times(dev, iters):
    """us per launch; our two forms with bias + residual + ReLU in the kernel, cuDNN fp16 the convolution with bias only."""
    import cutie_b200.kernels as K_
    out = []
    g = torch.Generator().manual_seed(5)
    bench_flag = torch.backends.cudnn.benchmark
    torch.backends.cudnn.benchmark = True                  # cuDNN's best fp16 algorithm, as an autotuned reference run
    try:
        with torch.inference_mode():
            for name, NB, Cin, Cout, H, W, k, cl in LAYERS:
                x = torch.randn(NB, Cin, H, W, generator=g).to(dev)
                z = torch.randn(NB, Cout, H, W, generator=g).to(dev)
                if cl:
                    x, z = x.contiguous(memory_format=torch.channels_last), z.contiguous(memory_format=torch.channels_last)
                w = (torch.randn(Cout, Cin, k, k, generator=g) * 0.02).to(dev)
                b = torch.randn(Cout, generator=g).to(dev)
                img32, img16 = K_.conv_weight_image(w), K_.conv_weight_image_f16(w)
                cnt = torch.zeros(8192, dtype=torch.int32, device=dev)
                xh, wh, bh = x.half(), w.half().contiguous(memory_format=torch.channels_last if cl else torch.contiguous_format), b.half()
                t32 = _timed(lambda: K_.conv_tc(x, img32, b, Cout, ksize=k, residual=z, relu_out=True, counters=cnt), iters)
                t16 = _timed(lambda: K_.conv_tc_f16(x, img16, b, Cout, ksize=k, residual=z, relu_out=True, counters=cnt), iters)
                tcd = _timed(lambda: F.conv2d(xh, wh, bh, padding=k // 2), iters)
                flops = 2.0 * NB * H * W * Cout * Cin * k * k
                out.append({'layer': name, 'conv_tc_3xtf32_us': t32, 'conv_tc_f16_us': t16, 'cudnn_fp16_us': tcd,
                            'conv_tc_f16_tflops': flops / t16 / 1e6})
                log(f'[layers] {out[-1]}')
    finally:
        torch.backends.cudnn.benchmark = bench_flag
    return out


def amp_parity(proc, cfg, frame, dev):
    """bench.parity_check's comparison for an amp step: the CPU oracle (fp32) re-computes one frame from the live state
    and the segment() logits are compared.  Without bench.parity_check's top-k reconciliation: the amp step's keys come
    from fp16-operand convolutions, so its top-k sets legitimately differ from the fp32 oracle's -- that difference is
    part of what amp costs, and is reported, not adopted."""
    from oracle.cpu_core import OracleCore
    from oracle.state_sync import export_state_to_oracle
    oc = export_state_to_oracle(proc, OracleCore(bench.make_net(cfg), cfg))
    graphs, proc.use_cuda_graphs = proc.use_cuda_graphs, False
    try:
        with torch.inference_mode():
            with torch.autocast('cuda', dtype=torch.float16):
                proc.step(frame.to(dev))
            torch.cuda.synchronize(dev)
            threads = torch.get_num_threads()
            torch.set_num_threads(bench.usable_cpus())
            oc.step(frame)
            torch.set_num_threads(threads)
    finally:
        proc.use_cuda_graphs = graphs
    diff = (proc.last_logits.cpu() - oc.last_logits).abs()
    return {'max_abs_logit_diff': float(diff.max()), 'mean_abs_logit_diff': float(diff.mean()),
            'memory_tokens': proc.memory.work_mem.size(0),
            'what': 'one amp frame after the timed blocks vs oracle/cpu_core.py (fp32) from the same live state, no '
                    'top-k reconciliation'}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=30, help='steps per timed block')
    ap.add_argument('--warmup', type=int, default=11, help='untimed steps per mode before the first block')
    ap.add_argument('--blocks', type=int, default=3, help='timed blocks per mode (alternating)')
    ap.add_argument('--iters', type=int, default=40, help='launches per layer timing')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('amp_bench.py needs a CUDA device')
    import cutie_b200.kernels as K_
    from cutie_b200.inference.inference_core import InferenceCore
    from cutie_b200.utils.synth import synthetic_video
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    hw = hardware()
    log(f'[hardware] {hw}')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = False
    wl = bench.WORKLOADS['cfg2']
    cfg = bench.make_cfg(wl)
    net = bench.make_net(cfg).to(dev).optimize_for_inference()
    K, B = args.steps, args.blocks
    n_frames = 2 * args.warmup + 2 * B * K + 2 * K + 8
    frames, mask = synthetic_video(n_frames, wl['H'], wl['W'], wl['K'], seed=0)
    objs = list(range(1, wl['K'] + 1))
    proc = InferenceCore(net, cfg=cfg, use_cuda_graphs=True)
    with torch.inference_mode():
        proc.step(frames[0].to(dev), mask.to(dev), objects=objs)
        for key, shr, vals in bench.synthetic_bank_chunks(wl):
            proc.memory.work_mem.add(key.to(dev), {o: vals[:, i].to(dev) for i, o in enumerate(objs)},
                                     shr.to(dev), None, as_permanent='no')
    n_tokens = proc.memory.work_mem.size(0)
    frames_dev = frames.to(dev)
    t = 1

    def run(steps, amp):
        nonlocal t
        with torch.inference_mode(), torch.autocast('cuda', dtype=torch.float16, enabled=amp):
            for _ in range(steps):
                proc.step(frames_dev[t])
                t += 1

    for amp in (False, True):                       # every graph variant of both modes is captured before timing
        run(args.warmup, amp)
    torch.cuda.synchronize()
    blocks = {'fp32': [], 'amp': []}
    for _ in range(B):
        for mode in ('fp32', 'amp'):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run(K, mode == 'amp')
            e1.record()
            torch.cuda.synchronize()
            blocks[mode].append(e0.elapsed_time(e1) / K)
            log(f'[block] {mode}: {blocks[mode][-1]:.3f} ms/step')
    # conv_tc kernel time per step: one eager block per mode, every C-ABI call between CUDA events
    conv = {}
    proc.use_cuda_graphs = False
    try:
        for mode in ('fp32', 'amp'):
            K_.PROFILE = []
            run(K, mode == 'amp')
            torch.cuda.synchronize()
            prof, K_.PROFILE = K_.PROFILE, None
            ms = [a.elapsed_time(b) for name, a, b in prof if name in ('conv_tc', 'conv_tc_f16')]
            conv[mode] = {'conv_tc_ms_per_step': sum(ms) / K, 'launches_per_step': len(ms) / K,
                          'f16_launches_per_step': sum(1 for p in prof if p[0] == 'conv_tc_f16') / K}
            log(f'[conv per step] {mode}: {conv[mode]}')
    finally:
        K_.PROFILE = None
        proc.use_cuda_graphs = True
    layers = layer_times(dev, args.iters)
    try:
        parity = amp_parity(proc, cfg, frames[t], dev)
    except Exception as e:                                 # noqa: BLE001 -- reported in the line, never hidden
        parity = {'error': f'{type(e).__name__}: {e}'[:300]}
    fps = {m: 1e3 / (sum(v) / len(v)) for m, v in blocks.items()}
    bench.emit({'what': 'InferenceCore.step fp32 vs fp16 autocast, bench.py cfg2 stream', 'hardware': hw,
                'workload': wl['desc'], 'memory_tokens': n_tokens, 'steps_per_block': K, 'blocks_per_mode': B,
                'frames_per_s': fps, 'ms_per_step_blocks': blocks, 'amp_over_fp32': fps['amp'] / fps['fp32'],
                'conv_tc_per_step': conv, 'layers_us': layers, 'parity_amp': parity,
                'epilogues': net.conv_epilogues.report()})


if __name__ == '__main__':
    main()
