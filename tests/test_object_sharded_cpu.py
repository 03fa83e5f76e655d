"""Object sharding (cutie_b200/inference/object_shards.py) on the CPU: the ownership rule, and whole streams over gloo
process groups of 2 and 3 ranks with the kernels emulated by tests/cpu_kernels.py (plus the two split aux-mask entries,
emulated below).  Every rank's result must be the same bits and track the un-sharded processor."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import object_shard_case
from tests.conftest import ROOT


# -- emulations of cutie_qt_mask_logits / cutie_qt_aux_fg (the same math as cpu_kernels.qt_aux_mask) ------------------
def qt_mask_logits(pixel, w, b, B, K):
    BK, E, HW = pixel.shape
    return ((torch.relu(pixel) * w.view(1, E, 1)).sum(1) + b).view(B, K, HW)


def qt_aux_fg(logits, positions):
    B, K, HW = logits.shape
    p = logits.sigmoid()
    bg = torch.prod(1 - p, dim=1, keepdim=True)
    allp = torch.cat([bg, p], 1).clamp(1e-7, 1 - 1e-7)
    lg = torch.log(allp / (1 - allp))
    fg = (lg[:, 1:] >= lg.max(1, keepdim=True)[0])[:, positions.long()]
    return fg.to(torch.uint8), fg.reshape(-1, HW).sum(1).int()


def _install():
    from tests import cpu_kernels as ck
    import cutie_b200.kernels as K_
    ck.install()
    K_.qt_mask_logits, K_.qt_aux_fg = qt_mask_logits, qt_aux_fg


def test_split_aux_emulation_matches_fused_emulation():
    from tests import cpu_kernels as ck
    g = torch.Generator().manual_seed(0)
    B, K, HW = 2, 5, 37
    pix = torch.randn(B * K, 256, HW, generator=g)
    w, b = torch.randn(256, generator=g) * 0.1, torch.randn(1, generator=g)
    lg, fg, cnt = ck.qt_aux_mask(pix, w, b, B, K)
    pos = torch.tensor([3, 0, 4], dtype=torch.int32)
    lg2 = qt_mask_logits(pix, w, b, B, K)
    fg2, cnt2 = qt_aux_fg(lg2, pos)
    assert torch.equal(lg, lg2)
    assert torch.equal(fg[:, pos.long()], fg2)
    assert torch.equal(cnt.view(B, K)[:, pos.long()].reshape(-1), cnt2)


# -- ownership ---------------------------------------------------------------------------------------------------------
class _Fake:
    """get_world_size / get_rank for one simulated rank (the table needs no collective)."""

    def __init__(self, world, rank):
        self.world, self.rank = world, rank

    def __enter__(self):
        self.orig = dist.get_world_size, dist.get_rank
        dist.get_world_size, dist.get_rank = (lambda g=None: self.world), (lambda g=None: self.rank)

    def __exit__(self, *exc):
        dist.get_world_size, dist.get_rank = self.orig


def _replay(world, rank, calls):
    from cutie_b200.inference.object_shards import ObjectShards
    with _Fake(world, rank):
        sh = ObjectShards(object())
    live, tables = [], []
    for op, ids in calls:
        if op == 'add':
            live += [o for o in ids if o not in live]
            sh.add(live)
        else:
            live = [o for o in live if o not in ids]
            sh.retain(live)
        tables.append(dict(sh.owner))
    return sh, tables


@pytest.mark.parametrize('world', [1, 2, 3, 4])
def test_ownership_is_balanced_stable_and_the_same_on_every_rank(world):
    calls = [('add', [1, 2, 3]), ('add', [4]), ('add', [5, 6, 7, 8, 9]), ('del', [2, 5]), ('add', [10]),
             ('add', [2]), ('del', [1, 3, 4]), ('add', [11, 12])]
    runs = [_replay(world, r, calls) for r in range(world)]
    tables = runs[0][1]
    for _, t in runs[1:]:
        assert t == tables                                   # every rank computes the same table
    for before, after in zip(tables, tables[1:]):            # an object never moves
        assert all(after[o] == r for o, r in before.items() if o in after)
    for t in tables[:3]:                                     # no deletions yet: balanced within one object
        load = [list(t.values()).count(r) for r in range(world)]
        assert max(load) - min(load) <= 1
    # without deletions the rule deals round-robin (ties go to the lowest rank)
    assert [tables[2][o] for o in range(1, 10)] == [i % world for i in range(9)]
    # after deleting 2 and 5, the freed ranks (least loaded) take the next objects; the re-added id 2 is a new placement
    t3, t4 = tables[3], tables[4]
    load3 = [list(t3.values()).count(r) for r in range(world)]
    assert t4[10] == load3.index(min(load3))
    assert 2 in tables[5] and 2 not in tables[3]
    # local lists and the group's positions follow the list order
    for sh, _ in runs:
        ids = sorted(sh.owner)
        grp = sh.group_of(ids)
        assert grp.local_ids == sh.local(ids) == [o for o in ids if sh.owner[o] == sh.rank]
        assert [ids[j] for j in grp.positions] == grp.local_ids


def test_fewer_objects_than_ranks_leaves_ranks_empty():
    sh, _ = _replay(4, 3, [('add', [7, 9])])
    assert sh.owner == {7: 0, 9: 1}
    assert sh.group_of([7, 9]).local_ids == []


def test_object_sharding_rejects_what_it_does_not_cover():
    from cutie_b200.config import default_config
    from cutie_b200.inference.inference_core import InferenceCore
    g = object()
    with pytest.raises(ValueError):
        InferenceCore(None, default_config(), object_shard_group=g, memory_shard_group=g)
    with pytest.raises(NotImplementedError):
        InferenceCore(None, default_config(chunk_size=2), object_shard_group=g)
    with pytest.raises(NotImplementedError):
        InferenceCore(None, default_config(save_aux=True), object_shard_group=g)


# -- gloo streams ------------------------------------------------------------------------------------------------------
def _cfg(kind):
    from cutie_b200.config import default_config
    if kind == 'long':
        return default_config(mem_every=1, use_long_term=True,
                              long_term=dict(max_mem_frames=4, min_mem_frames=2, num_prototypes=8, max_num_tokens=40,
                                             buffer_tokens=10))
    return default_config(mem_every=2, max_mem_frames=3, flip_aug=(kind == 'flip'))


CASES = {
    # name: (config, run() keywords).  The foreground test and top-k are discrete: a pixel whose decision is tied to
    # within the rounding that differs between batch sizes flips and moves the next frames' logits by ~1e-2 (DESIGN.md
    # section 4).  The long-term clip uses a seed without such a tie (seed 3 has one on its last frame).
    'fifo': ('fifo', dict(T=9)),
    'long': ('long', dict(T=13, seed=4)),
    'flip': ('flip', dict(T=7)),
    'few': ('fifo', dict(T=6, K0=1, extra=0, delete=())),
}


def _stream_worker(rank, world, port, case, ret):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        _install()
        from cutie_b200.model.cutie import CUTIE
        from oracle.synth import synthetic_state_dict
        from tests import object_shard_case
        torch.set_num_threads(2)
        kind, kw = CASES[case]
        cfg = _cfg(kind)
        net = CUTIE(cfg).eval()
        net.load_state_dict(synthetic_state_dict(net.state_dict(), 0))
        ret[rank] = object_shard_case.run(net, cfg, 'cpu', dist.group.WORLD, **kw)
    finally:
        dist.destroy_process_group()


STREAMS = [(2, 'fifo'), (3, 'fifo'), (2, 'long'), (3, 'long'), (2, 'flip'), (3, 'few')]


@pytest.mark.parametrize('world,case', STREAMS)
def test_object_sharded_stream_matches_unsharded(world, case):
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_stream_worker, args=(world, object_shard_case.free_port(), case, ret), nprocs=world, join=True)
    res = [ret[r] for r in range(world)]
    for r, x in enumerate(res):
        assert x['finite'], f'rank {r}: non-finite prob or logits'
        # The ranks compute the replicated part of a step (the segment tail, the mask merge, the soft aggregation of an
        # input mask) from bit-identical inputs.  ATen's CPU float kernels do not promise bit-reproducible results across
        # processes, though: a loaded host once gave the two ranks of a 2-rank stream different bits on frame 0 -- the
        # soft aggregation of the input mask, which no exchange touches -- in 44 496 near-zero probabilities, at most
        # 1.4e-19 apart.  So the CPU bar is 1e-12, far below any exchange or ownership error (those move whole objects'
        # planes); the CUDA kernels are deterministic and tests/test_gpu_object_sharded.py holds the ranks to every bit.
        assert x['cross_rank'] <= 1e-12, \
            f'rank {r}: prob differs between ranks by {x["cross_rank"]}; first (frame, elements, max |diff|) {x["mismatch"]}'
        assert x['owned'], f'rank {r}: holds values / sensory / summaries of objects it does not own'
        assert x['worst'] < 2e-4, f'rank {r}: sharded stream deviates by {x["worst"]}'
        assert x['owners'] == res[0]['owners']
    if case != 'few':
        assert sorted(res[0]['buckets']) == [2, 4] and 2 not in res[0]['live']       # second bucket, one deletion
    else:
        assert len(res[0]['owners'][-1]) < world
    if case == 'long':
        trace = res[0]['long_trace']
        assert max(trace) == 32 and any(a > b for a, b in zip(trace, trace[1:])), \
            f'the clip must consolidate and remove obsolete features: {trace}'


def test_idle_rank_joins_every_foreground_exchange(cpu_kernels, monkeypatch):
    """A rank that owns none of a bucket's objects must make exactly the all-gathers QueryTransformer.forward makes,
    with the same shapes, or the ranks' collectives fall out of step."""
    from cutie_b200.config import default_config
    from cutie_b200.model.object_transformer import QueryTransformer
    import cutie_b200.kernels as K_
    monkeypatch.setattr(K_, 'qt_mask_logits', qt_mask_logits)
    monkeypatch.setattr(K_, 'qt_aux_fg', qt_aux_fg)

    class Recorder:
        def __init__(self, n_local):
            self.calls, self.n = [], n_local

        def gather(self, x):
            self.calls.append((x.shape[0], x.shape[2]))
            return x.new_zeros(x.shape[0], 3, x.shape[2])

        def positions_tensor(self, device):
            return torch.arange(self.n, dtype=torch.int32)

    cfg = default_config()
    qt = QueryTransformer(cfg.model).eval()
    B, K, E, h, w = 1, 2, cfg.model.embed_dim, 4, 6
    busy, idle = Recorder(K), Recorder(0)
    with torch.inference_mode():
        qt(torch.randn(B, K, E, h, w), torch.rand(B, K, 1, qt.num_queries, E + 1), objects=busy)
        qt.exchange_without_objects(idle, B, h * w, 'cpu')
    assert len(busy.calls) == qt.num_blocks + 1 and idle.calls == busy.calls


def test_split_aux_entries_validate_arguments_on_the_host():
    """cutie_qt_mask_logits / cutie_qt_aux_fg reject null pointers, empty sizes and more positions than objects before
    any CUDA call."""
    import ctypes
    import __graft_entry__ as ge
    from cutie_b200 import kernels
    ge.build()
    lib = kernels.lib()
    one = ctypes.c_void_p(0x1000)                      # never dereferenced: validation fails first
    i64 = ctypes.c_int64
    ml = lib.cutie_qt_mask_logits
    assert ml(None, one, one, i64(1), i64(2), i64(256), i64(10), one, None) == -1
    assert b'cutie_qt_mask_logits' in lib.cutie_b200_last_error()
    assert ml(one, one, one, i64(1), i64(2), i64(128), i64(10), one, None) == -1          # embed_dim != 256
    assert ml(one, one, one, i64(1), i64(0), i64(256), i64(10), one, None) == -1          # no objects
    fg = lib.cutie_qt_aux_fg
    assert fg(one, None, i64(1), i64(2), i64(1), i64(10), one, one, None) == -1
    assert b'cutie_qt_aux_fg' in lib.cutie_b200_last_error()
    assert fg(one, one, i64(1), i64(2), i64(3), i64(10), one, one, None) == -1            # n > K
    assert b'more positions' in lib.cutie_b200_last_error()
    assert fg(one, one, i64(1), i64(2), i64(0), i64(10), one, one, None) == -1            # n == 0
    assert fg(one, one, i64(1), i64(2), i64(1), i64(0), one, one, None) == -1             # HW == 0
