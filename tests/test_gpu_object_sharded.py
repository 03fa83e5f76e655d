"""Object sharding on the GPU: the split aux-mask entries (cutie_qt_mask_logits + cutie_qt_aux_fg) against the fused
cutie_qt_aux_mask, an object-sharded stream over a one-rank NCCL group against the plain processor (every exchange is an
identity there, so every bit must agree), and on >= 2 GPUs a 480p stream sharded over all of them."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import object_shard_case
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def K_():
    import __graft_entry__ as ge
    if not os.path.exists(ge.LIB):
        ge.build()
    import cutie_b200.kernels as k
    k.lib()
    return k


def _inputs(B, K, HW, seed):
    g = torch.Generator().manual_seed(seed)
    pix = torch.randn(B, K, 256, HW, generator=g)
    w = torch.randn(256, generator=g) * 0.1
    b = torch.randn(1, generator=g) * 0.5
    if K >= 2:                      # object 0 foreground everywhere, object 1 nowhere
        pix[:, 0] = 40.0 * (w > 0).float().view(256, 1)
        pix[:, 1] = 40.0 * (w < 0).float().view(256, 1)
    return pix, w, b


def _position_lists(K):
    lists = [list(range(K)), [K - 1]]
    if K >= 3:
        lists += [list(range(0, K, 2)), list(range(K - 1, 0, -3)), [1, 0]]
    return lists


@pytest.mark.parametrize('B', [1, 2])
@pytest.mark.parametrize('K', [1, 2, 3, 15, 16, 17, 32, 33, 48])
@pytest.mark.parametrize('HW', [1620, 37])
def test_split_aux_mask_equals_fused(K_, B, K, HW):
    pix, w, b = _inputs(B, K, HW, seed=K * 7 + B + HW)
    pix, w, b = pix.cuda(), w.cuda(), b.cuda()
    lg, fg, cnt = K_.qt_aux_mask(pix.reshape(B * K, 256, HW), w, b, B, K)
    cnt = cnt.view(B, K)
    if K >= 2:
        assert bool((cnt[:, 0] == HW).all()) and bool((cnt[:, 1] == 0).all())
    assert torch.equal(K_.qt_mask_logits(pix.reshape(B * K, 256, HW), w, b, B, K), lg)
    for pos in _position_lists(K):
        # a rank's pixel tensor holds its own objects only
        local = pix[:, pos].reshape(B * len(pos), 256, HW).contiguous()
        assert torch.equal(K_.qt_mask_logits(local, w, b, B, len(pos)), lg[:, pos])
        p = torch.tensor(pos, dtype=torch.int32, device='cuda')
        fg2, cnt2 = K_.qt_aux_fg(lg, p)
        assert torch.equal(fg2, fg[:, pos]), pos
        assert torch.equal(cnt2.view(B, len(pos)), cnt[:, pos]), pos
    torch.cuda.synchronize()


def _init(rank, world, port):
    sys.path.insert(0, ROOT)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=torch.device('cuda', rank))
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def _cfg(kind):
    from cutie_b200.config import default_config
    if kind == 'long':
        return default_config(mem_every=1, use_long_term=True,
                              long_term=dict(max_mem_frames=4, min_mem_frames=2, num_prototypes=16, max_num_tokens=60,
                                             buffer_tokens=20))
    return default_config(mem_every=2, max_mem_frames=4)


def _net(cfg, dev):
    """The product's model: synthetic weights, optimize_for_inference (folded trunks, fused epilogues and glue)."""
    from cutie_b200.model.cutie import CUTIE
    from cutie_b200.utils.synth import synthetic_state_dict
    net = CUTIE(cfg).eval()
    net.load_state_dict(synthetic_state_dict(net.state_dict(), 0))
    return net.to(dev).optimize_for_inference()


def _world1_worker(rank, world, port, kind, ret):
    _init(rank, world, port)
    try:
        from tests import object_shard_case
        cfg = _cfg(kind)
        dev = torch.device('cuda', rank)
        out = object_shard_case.run(_net(cfg, dev), cfg, dev, dist.group.WORLD, T=10, H=240, W=432, K0=5, extra=2,
                                    add_at=3, delete_at=6, delete=(2, 6))
        torch.cuda.synchronize()
        ret[rank] = out
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize('kind', ['fifo', 'long'])
def test_world1_object_sharding_is_bit_identical_to_plain(kind):
    """A one-rank group: every gather and the broadcast are identities and the batches are the same, so the sharded
    processor's prob and last_logits must equal the plain processor's bit for bit on every frame."""
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_world1_worker, args=(1, object_shard_case.free_port(), kind, ret), nprocs=1, join=True)
    x = ret[0]
    assert x['finite'], 'non-finite prob or logits'
    assert x['worst'] == 0.0, f'sharded and plain differ by {x["worst"]}'
    assert x['same'] and x['owned']
    assert sorted(x['buckets']) == [1, 4]


def _multi_worker(rank, world, port, kind, ret):
    _init(rank, world, port)
    try:
        from tests import object_shard_case
        cfg = _cfg(kind)
        dev = torch.device('cuda', rank)
        out = object_shard_case.run(_net(cfg, dev), cfg, dev, dist.group.WORLD, T=8, H=480, W=864, K0=10, extra=2,
                                    add_at=3, delete_at=5, delete=(4,))
        torch.cuda.synchronize()
        ret[rank] = out
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs >= 2 GPUs')
@pytest.mark.parametrize('kind', ['fifo', 'long'])
def test_object_sharded_480p_stream_nccl(kind):
    """12 objects (10, then 2 more in a second bucket, then one deleted) at 480p sharded over every GPU: the same prob on
    every rank, logits within 2e-4 of the single-GPU un-sharded run, values held by their owners only."""
    world = min(torch.cuda.device_count(), 8)
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_multi_worker, args=(world, object_shard_case.free_port(), kind, ret), nprocs=world, join=True)
    for r in range(world):
        x = ret[r]
        assert x['finite'], f'rank {r}: non-finite prob or logits'
        assert x['same'], f'rank {r}: prob differs between ranks at (frame, elements, max |diff|) = {x["mismatch"]}'
        assert x['owned'], f'rank {r}: holds values of objects it does not own'
        assert x['logit_diff'] < 2e-4, f'rank {r}: logits deviate by {x["logit_diff"]}'
