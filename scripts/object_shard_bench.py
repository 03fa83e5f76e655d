"""Object sharding: InferenceCore.step on one synthetic 480p stream with its objects split over the GPUs of a node.

    torchrun --nproc_per_node=G scripts/object_shard_bench.py [--objects 8,16,32,48] [--steps S] [--blocks B]
    python scripts/object_shard_bench.py ...            (one GPU: a one-rank group)

One JSON line on stdout (rank 0).  Per object count K, in one call and alternated block by block:
* `sharded`: the object-sharded processor on all G ranks (eager: the segment and mask-encoder graphs are off under object
  sharding).  ms/step over timed blocks of S steps, each ending in a device synchronise on every rank and a barrier
  (the median block, the mean and every block are reported);
  then one profiled block in which every exchange (the key broadcast and the logits all-gathers) is bracketed by CUDA
  events: exchange ms/step and calls/step, and the largest over the ranks;
* `plain_eager` / `plain_graphs`: the un-sharded processor on rank 0's GPU alone, eager and with CUDA graphs (the other
  ranks wait at a barrier).
Stream, weights and memory settings are scripts/objects_bench.py's: bench.py's synthetic 480p video and weights, the
optimised model, a 6-frame working memory (mem_every 5) filled during the warm-up.  The card's name and power limit are
read in the same call.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import bench  # noqa: E402  (points fd 1 at stderr; bench.emit writes the JSON line to the real stdout)
from scripts.objects_bench import H, W, hardware  # noqa: E402

log = bench.log


class ExchangeTimer:
    """Brackets ObjectShards.broadcast and ObjectGroup.gather with CUDA events while `on`."""

    def __init__(self):
        from cutie_b200.inference import object_shards as S
        self.S, self.on, self.marks = S, False, []
        self.orig = S.ObjectShards.broadcast, S.ObjectGroup.gather
        timer = self

        def timed(fn):
            def wrapper(*a, **kw):
                if not timer.on:
                    return fn(*a, **kw)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                out = fn(*a, **kw)
                e1.record()
                timer.marks.append((e0, e1))
                return out
            return wrapper
        S.ObjectShards.broadcast, S.ObjectGroup.gather = timed(self.orig[0]), timed(self.orig[1])

    def take(self):
        ms = [a.elapsed_time(b) for a, b in self.marks]
        self.marks = []
        return sum(ms), len(ms)


class Stream:
    def __init__(self, net, cfg, K, frames, mask, **kw):
        from cutie_b200.inference.inference_core import InferenceCore
        self.frames, self.mask, self.K, self.dev, self.t = frames, mask, K, frames.device, 0
        self.proc = InferenceCore(net, cfg=cfg, **kw)

    def run(self, n):
        with torch.inference_mode():
            for _ in range(n):
                if self.t == 0:
                    self.proc.step(self.frames[0], self.mask.to(self.dev), objects=list(range(1, self.K + 1)))
                else:
                    self.proc.step(self.frames[self.t])
                self.t += 1

    def block(self, steps, group=None):
        """ms/step of `steps` steps, ending in a device synchronise (and a barrier over `group`)."""
        t0 = time.perf_counter()
        self.run(steps)
        torch.cuda.synchronize()
        if group is not None:
            dist.barrier(group=group)
        return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--objects', default='8,16,32,48')
    ap.add_argument('--steps', type=int, default=10, help='steps per timed block')
    ap.add_argument('--blocks', type=int, default=3, help='timed blocks per processor and object count')
    ap.add_argument('--warmup', type=int, default=30, help='untimed steps first (fills the working memory)')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('object_shard_bench.py needs a CUDA device')
    if 'RANK' not in os.environ:                     # plain `python`: a one-rank group
        os.environ.update(RANK='0', WORLD_SIZE='1', LOCAL_RANK='0', MASTER_ADDR='127.0.0.1', MASTER_PORT='29533')
    local = int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    dist.init_process_group('nccl', device_id=dev)
    rank, world = dist.get_rank(), dist.get_world_size()
    try:
        from cutie_b200.config import default_config
        from cutie_b200.utils.synth import synthetic_video
        hw = hardware()
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        torch.backends.cudnn.benchmark = False
        cfg = default_config(mem_every=5, max_mem_frames=6, use_long_term=False, top_k=30)
        net = bench.make_net(cfg).to(dev).optimize_for_inference()
        timer = ExchangeTimer()
        n_frames = args.warmup + 2 * args.blocks * args.steps + args.steps + 1
        rows = []
        for K in [int(k) for k in args.objects.split(',') if k]:
            frames, mask = synthetic_video(n_frames, H, W, K, seed=0)
            frames = frames.to(dev)
            sharded = Stream(net, cfg, K, frames, mask, object_shard_group=dist.group.WORLD)
            plain = {name: Stream(net, cfg, K, frames, mask, use_cuda_graphs=g) if rank == 0 else None
                     for name, g in (('plain_eager', False), ('plain_graphs', True))}
            sharded.run(args.warmup)
            for p in plain.values():
                if p is not None:
                    p.run(args.warmup)
            torch.cuda.synchronize()
            dist.barrier()
            ms = {'sharded': [], 'plain_eager': [], 'plain_graphs': []}
            for _ in range(args.blocks):
                ms['sharded'].append(sharded.block(args.steps, dist.group.WORLD))
                for name, p in plain.items():
                    if p is not None:
                        ms[name].append(p.block(args.steps))
                dist.barrier()
            timer.on = True
            sharded.block(args.steps, dist.group.WORLD)
            timer.on = False
            ex_ms, ex_calls = timer.take()
            ex = torch.tensor([ex_ms / args.steps], device=dev)
            allex = [torch.zeros_like(ex) for _ in range(world)]
            dist.all_gather(allex, ex)
            owned = torch.tensor([len(sharded.proc.object_shards.local(sharded.proc.object_manager.all_obj_ids))],
                                 device=dev)
            dist.all_reduce(owned, op=dist.ReduceOp.MAX)
            row = {'objects': K, 'world': world, 'max_objects_per_rank': int(owned),
                   'exchange_ms_per_step': [float(e) for e in allex], 'exchange_calls_per_step': ex_calls / args.steps}
            for name, v in ms.items():
                if v:
                    row[name] = {'ms_per_step_median': sorted(v)[len(v) // 2], 'ms_per_step_mean': sum(v) / len(v),
                                 'ms_per_step_blocks': v}
            rows.append(row)
            if rank == 0:
                log(f'[object-shard] {row}')
            del sharded, plain
            torch.cuda.empty_cache()
        if rank == 0:
            bench.emit({'what': 'InferenceCore.step with objects sharded over the GPUs vs un-sharded on one GPU, '
                                'synthetic 480p stream, optimised model', 'hardware': hw, 'world': world,
                        'steps_per_block': args.steps, 'blocks': args.blocks, 'warmup': args.warmup, 'rows': rows})
    finally:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
