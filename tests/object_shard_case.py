"""One video stream run twice on every rank of a process group -- object-sharded over the group and un-sharded -- frame by
frame on the same inputs.  Shared by the gloo streams (tests/test_object_sharded_cpu.py, kernels emulated) and the NCCL
streams (tests/test_gpu_object_sharded.py).

The stream: `K0` objects on frame 0 (one bucket), `extra` more on frame `add_at` (a second bucket), the objects
`delete` removed before frame `delete_at`."""
import torch
import torch.distributed as dist


def free_port() -> int:
    """A port no process listens on now (the OS picks it), so no two process groups share a rendezvous."""
    import socket
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        return sk.getsockname()[1]


def _extra_mask(H, W, first_id, n):
    m = torch.zeros(H, W, dtype=torch.int64)
    y0, y1 = int(H * 0.72), int(H * 0.92)
    for j in range(n):
        x0 = int(W * (0.05 + 0.9 * j / max(n, 1)))
        m[y0:y1, x0:x0 + max(W // (2 * n + 2), 2)] = first_id + j
    return m


def holds_only_owned(proc) -> bool:
    """Value arrays, sensory state and object summaries of the live objects exist on the owning rank only."""
    sh, mem = proc.object_shards, proc.memory
    live = proc.object_manager.all_obj_ids
    for o in live:
        mine = sh.owner[o] == sh.rank
        if (o in mem.sensory) != mine or (o in mem.obj_v) != mine:
            return False
    stores = [mem.work_mem] + ([mem.long_mem] if mem.use_long_term else [])
    for store in stores:
        for bk in store._b.values():
            for o in bk.objects:
                mine = sh.owner[o] == sh.rank
                for arena in (bk.perm, bk.temp):
                    if arena.widths and (('val', o) in arena.widths) != mine:
                        return False
    return True


def _diff(a: torch.Tensor, b: torch.Tensor) -> float:
    """max |a - b|, inf where either holds a NaN or an inf (a Python max over floats would drop a NaN)."""
    return float(torch.nan_to_num((a - b).abs(), nan=float('inf')).max())


def run(net, cfg, device, group, *, T=9, H=96, W=160, K0=5, extra=2, add_at=3, delete_at=5, delete=(2,), seed=3):
    """Returns dict(worst / logit_diff = max |sharded - plain| over prob and last_logits / last_logits alone (inf if
    either run gives a non-finite value), finite = every prob and last_logits of both runs is finite, same = prob
    bit-identical on every rank at every frame, mismatch = None or (frame, elements, max |difference|) of the first frame
    whose prob differs between ranks, cross_rank = max |difference| between the ranks' prob over all frames, owned = holds_only_owned at every frame, owners = the ownership table after each
    frame, long_trace = the un-sharded run's long-term token count of bucket 0 after each frame)."""
    from cutie_b200.inference.inference_core import InferenceCore
    from cutie_b200.utils.synth import synthetic_video
    world = dist.get_world_size(group)
    frames, mask = synthetic_video(T, H, W, K0, seed=seed)
    add = _extra_mask(H, W, K0 + 1, extra) if extra else None
    sharded = InferenceCore(net, cfg=cfg, object_shard_group=group)
    plain = InferenceCore(net, cfg=cfg)
    worst, logit_diff, finite, mismatch, cross_rank, owned, owners, long_trace = 0.0, 0.0, True, None, 0.0, True, [], []
    with torch.inference_mode():
        for ti in range(T):
            if ti == delete_at and delete:
                sharded.delete_objects(list(delete))
                plain.delete_objects(list(delete))
            if ti == 0:
                args, kw = (frames[0].to(device), mask.to(device)), dict(objects=list(range(1, K0 + 1)))
            elif ti == add_at and add is not None:
                args, kw = (frames[ti].to(device), add.to(device)), dict(objects=list(range(K0 + 1, K0 + extra + 1)))
            else:
                args, kw = (frames[ti].to(device),), {}
            ps = sharded.step(*args, **kw)
            pp = plain.step(*args, **kw)
            finite = finite and bool(torch.isfinite(ps).all()) and bool(torch.isfinite(pp).all())
            worst = max(worst, _diff(ps, pp))
            if sharded.last_logits is not None and ti > 0:
                finite = finite and bool(torch.isfinite(sharded.last_logits).all())
                logit_diff = max(logit_diff, _diff(sharded.last_logits, plain.last_logits))
            # bit identity across ranks: compare the bits, not the values (NaN != NaN, -0.0 == 0.0)
            allp = torch.empty((world * ps.shape[0],) + tuple(ps.shape[1:]), dtype=ps.dtype, device=ps.device)
            dist.all_gather_into_tensor(allp, ps.contiguous(), group=group)
            allp = allp.view((world,) + tuple(ps.shape))
            bits = allp.view(torch.int32)
            differ = (bits != bits[:1]).any(0)
            if bool(differ.any()):
                spread = _diff(allp.amax(0), allp.amin(0))
                cross_rank = max(cross_rank, spread)
                if mismatch is None:
                    mismatch = (ti, int(differ.sum()), spread)
            owned = owned and holds_only_owned(sharded)
            owners.append(dict(sharded.object_shards.owner))
            lm = plain.memory.long_mem if plain.memory.use_long_term else None
            long_trace.append(lm.size(0) if lm is not None and lm.engaged(0) else 0)
    return dict(worst=max(worst, logit_diff), logit_diff=logit_diff, finite=finite, same=mismatch is None,
                mismatch=mismatch, cross_rank=cross_rank, owned=owned, owners=owners, live=list(sharded.object_manager.all_obj_ids),
                buckets=[len(v) for v in sharded.memory.work_mem.buckets.values()], long_trace=long_trace)
