"""Cost of the object count: InferenceCore.step on a synthetic 480p stream for K objects, one JSON line on stdout.

    python scripts/objects_bench.py [--objects 3,8,16,17,24,32,33,48] [--lt-objects 16,17,40] [--steps S] [--blocks B]

* hardware: the card's name and power limit (read-only nvidia-smi query), beside every number;
* FIFO stream, per K: bench.py's synthetic 480p video and weights (cutie_b200.utils.synth), optimised model, CUDA graphs,
  a 6-frame working memory (mem_every 5) filled during the warm-up.  Frames/s over B timed blocks of S steps, each block
  ending in a device synchronise; then one eager block with every C-ABI call between CUDA events gives the per-step
  kernel time of cutie_readout_gather and cutie_qt_aux_mask (and their launches per step);
* long-term stream, per K: the same with long-term memory (mem_every 1, 4..8 working frames, 128 prototypes), so
  consolidations fall inside the timed window; reports frames/s and the time of each cutie_consolidate call.
K = 17 and 33 are the first counts past one launch of the readout gather / consolidation (16 objects) and past the
register form of the aux-mask kernel (32 objects).
"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402  (points fd 1 at stderr; bench.emit writes the JSON line to the real stdout)

log = bench.log
H, W = 480, 854


def hardware():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    name, power = (r.stdout.strip().splitlines() or [','])[0].split(',')[:2]
    return {'name': name.strip(), 'power_limit': power.strip()}


def measure(net, cfg, K, steps, blocks, warmup, dev, profile_names):
    import cutie_b200.kernels as K_
    from cutie_b200.inference.inference_core import InferenceCore
    from cutie_b200.utils.synth import synthetic_video
    n_frames = warmup + blocks * steps + steps + 1
    frames, mask = synthetic_video(n_frames, H, W, K, seed=0)
    frames = frames.to(dev)
    proc = InferenceCore(net, cfg=cfg, use_cuda_graphs=True)
    t = 0

    def run(n):
        nonlocal t
        with torch.inference_mode():
            for _ in range(n):
                if t == 0:
                    proc.step(frames[0], mask.to(dev), objects=list(range(1, K + 1)))
                else:
                    proc.step(frames[t])
                t += 1

    run(warmup)
    torch.cuda.synchronize()
    ms = []
    for _ in range(blocks):
        t0 = time.perf_counter()
        run(steps)
        torch.cuda.synchronize()
        ms.append((time.perf_counter() - t0) * 1e3 / steps)
    # per-kernel time: one eager block, every C-ABI call bracketed by CUDA events
    proc.use_cuda_graphs = False
    K_.PROFILE = []
    try:
        run(steps)
        torch.cuda.synchronize()
        prof = K_.PROFILE
    finally:
        K_.PROFILE = None
    kern = {}
    for name in profile_names:
        times = [a.elapsed_time(b) for n, a, b in prof if n == name]
        kern[name] = {'ms_per_step': sum(times) / steps, 'calls_per_step': len(times) / steps,
                      'ms_per_call': (sum(times) / len(times)) if times else None}
    row = {'objects': K, 'frames_per_s': 1e3 / (sum(ms) / len(ms)), 'ms_per_step_blocks': ms, 'kernels': kern,
           'memory_tokens': proc.memory.work_mem.size(0)}
    if cfg.use_long_term:
        row['long_term_tokens'] = proc.memory.long_mem.size(0) if proc.memory.long_mem.engaged() else 0
    del proc
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--objects', default='3,8,16,17,24,32,33,48')
    ap.add_argument('--lt-objects', default='16,17,40')
    ap.add_argument('--steps', type=int, default=10, help='steps per timed block')
    ap.add_argument('--blocks', type=int, default=3, help='timed blocks per object count')
    ap.add_argument('--warmup', type=int, default=30, help='untimed steps first (fills the working memory)')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('objects_bench.py needs a CUDA device')
    from cutie_b200.config import default_config
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    hw = hardware()
    log(f'[hardware] {hw}')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = False
    fifo_cfg = default_config(mem_every=5, max_mem_frames=6, use_long_term=False, top_k=30)
    lt_cfg = default_config(mem_every=1, use_long_term=True, top_k=30,
                            long_term=dict(max_mem_frames=8, min_mem_frames=4, num_prototypes=128,
                                           max_num_tokens=10000, buffer_tokens=2000))
    fifo, lt = [], []
    net = bench.make_net(fifo_cfg).to(dev).optimize_for_inference()
    for K in [int(k) for k in args.objects.split(',') if k]:
        fifo.append(measure(net, fifo_cfg, K, args.steps, args.blocks, args.warmup, dev,
                            ('readout_gather', 'qt_aux_mask')))
        log(f'[fifo] {fifo[-1]}')
    for K in [int(k) for k in args.lt_objects.split(',') if k]:
        lt.append(measure(net, lt_cfg, K, args.steps, args.blocks, args.warmup, dev,
                          ('readout_gather', 'qt_aux_mask', 'consolidate')))
        log(f'[long-term] {lt[-1]}')
    bench.emit({'what': 'InferenceCore.step vs object count, synthetic 480p stream, optimised model, CUDA graphs',
                'hardware': hw, 'steps_per_block': args.steps, 'blocks': args.blocks, 'warmup': args.warmup,
                'fifo': fifo, 'long_term': lt})


if __name__ == '__main__':
    main()
