"""Videos with more objects than one launch of a per-object kernel takes: the readout gather and the consolidation
(16 objects per launch) and the register form of the aux-mask kernel (32 objects).

Kernel level: an object's output never depends on which other objects share the call -- every plane / row is the same
bits as a call with that object alone -- and the grouped results match the CPU emulation.  End to end: 20 and 40 objects
against the CPU oracle (teacher-forced, FIFO and long-term memory), CUDA graphs against the eager path, a second bucket
with deletions, and 20 objects free-running against the unmodified reference (tests/golden/e2e_many_objects.npz)."""
import os

import numpy as np
import pytest
import torch

from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def K_():
    import __graft_entry__ as ge
    if not os.path.exists(ge.LIB):
        ge.build()
    import cutie_b200.kernels as k
    k.lib()
    return k


def _segments(K_, key, shr, vals, cuts):
    from tests.test_gpu_kernels import segments_of
    return segments_of(K_, key, shr, vals, cuts)


def _only(K_, segs, ks):
    return [K_.BankSegment(s.key, s.shrinkage, tuple(s.values[k] for k in ks)) for s in segs]


# ---------------------------------------------------------------------------------------------
# readout gather
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [17, 33, 64])
@pytest.mark.parametrize('B,cuts', [(1, ()), (2, (100,)), (1, (40, 41, 200)), (2, (7, 150))])
def test_readout_gather_any_object_count(K_, K, B, cuts):
    from tests import cpu_kernels as ck
    from tests.test_gpu_kernels import make_bank
    N, Q, kpad = 260, 70, 32
    key, shr, vals = make_bank(B, N, K, seed=K + 10 * B + len(cuts))
    g = torch.Generator().manual_seed(K * 7 + B)
    idx = torch.randint(0, N, (B, Q, kpad), generator=g, dtype=torch.int32)
    w = torch.rand(B, Q, kpad, generator=g)
    holes = torch.rand(B, Q, kpad, generator=g) < 0.3            # sharded banks own a subset of the winners
    idx[holes] = -1
    w[holes] = 0
    segs = _segments(K_, key, shr, vals, cuts)
    idx_d, w_d = idx.cuda(), w.cuda()
    out = K_.readout_gather(idx_d, w_d, segs)
    for k in range(K):
        alone = K_.readout_gather(idx_d, w_d, _only(K_, segs, [k]))
        assert torch.equal(out[:, k], alone[:, 0]), k
    ref = ck.readout_gather(idx, w, [K_.BankSegment(key, shr, tuple(vals))])
    assert torch.allclose(out.cpu(), ref, rtol=1e-4, atol=2e-5)


# ---------------------------------------------------------------------------------------------
# consolidation
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('K', [17, 40])
@pytest.mark.parametrize('with_stats', [False, True])
def test_consolidate_any_object_count(K_, K, with_stats):
    from tests import cpu_kernels as ck
    from tests.test_gpu_kernels import make_bank
    B, N, P = 2, 300, 18                                          # P not a multiple of the 4 prototypes per CTA
    key, shr, vals = make_bank(B, N, K, seed=100 + K)
    g = torch.Generator().manual_seed(200 + K)
    pk = key[:, torch.randperm(N, generator=g)[:P]].contiguous()
    pe = torch.sigmoid(torch.randn(B, P, 64, generator=g))
    segs = _segments(K_, key, shr, vals, (77, 200))
    pk_d, pe_d = pk.cuda(), pe.cuda()

    def run(ks):
        ov = [torch.zeros(B, P, 256).cuda() for _ in ks]
        osr = torch.zeros(B, P).cuda()
        stats = (torch.zeros(B, P).cuda(), torch.zeros(B, P).cuda()) if with_stats else None
        K_.consolidate(_only(K_, segs, ks), pk_d, pe_d, ov, osr, stats=stats)
        return ov, osr, stats

    ov, osr, stats = run(list(range(K)))
    for k in range(K):
        alone, _, _ = run([k])
        assert torch.equal(ov[k], alone[0]), k
    ov16, osr16, stats16 = run(list(range(16)))
    assert torch.equal(osr, osr16)
    if with_stats:
        assert torch.equal(stats[0], stats16[0]) and torch.equal(stats[1], stats16[1])
    # CPU emulation (dense softmax of the oracle)
    rv = [torch.zeros(B, P, 256) for _ in range(K)]
    rs = torch.zeros(B, P)
    rstats = (torch.zeros(B, P), torch.zeros(B, P)) if with_stats else None
    ck.consolidate([K_.BankSegment(key, shr, tuple(vals))], pk, pe, rv, rs, stats=rstats)
    for k in range(K):
        assert torch.allclose(ov[k].cpu(), rv[k], rtol=1e-4, atol=2e-5), k
    assert torch.allclose(osr.cpu(), rs, rtol=1e-4, atol=2e-5)
    if with_stats:
        assert torch.allclose(stats[0].cpu(), rstats[0], rtol=1e-5, atol=1e-5)
        assert torch.allclose(stats[1].cpu(), rstats[1], rtol=1e-4, atol=1e-5)


# ---------------------------------------------------------------------------------------------
# aux mask
# ---------------------------------------------------------------------------------------------
def _aux_inputs(B, K, HW, seed):
    g = torch.Generator().manual_seed(seed)
    pix = torch.randn(B * K, 256, HW, generator=g) * 2
    w = torch.randn(256, generator=g) / 8
    b = torch.randn(1, generator=g)
    return pix, w, b


@pytest.mark.parametrize('K', [32, 33, 48, 64])
@pytest.mark.parametrize('B,HW', [(1, 1620), (2, 77)])
def test_qt_aux_mask_any_object_count(K_, B, K, HW):
    from tests import cpu_kernels as ck
    pix, w, b = _aux_inputs(B, K, HW, 7 + K)
    lc, fc, cc = ck.qt_aux_mask(pix, w, b, B, K)
    lg, fg, cg = K_.qt_aux_mask(pix.cuda(), w.cuda(), b.cuda(), B, K)
    assert torch.allclose(lg.cpu(), lc, rtol=1e-4, atol=1e-4)
    diff = (fg.cpu() != fc)
    if diff.any():           # the foreground bit may differ only where two log-odds are within rounding of each other
        p = lc.sigmoid()
        allp = torch.cat([torch.prod(1 - p, 1, keepdim=True), p], 1).clamp(1e-7, 1 - 1e-7)
        lo = torch.log(allp / (1 - allp))
        top2 = lo.topk(2, dim=1)[0]
        near = (top2[:, 0] - top2[:, 1]).abs() < 1e-4
        assert (diff.any(1) <= near).all()
    assert (cg.cpu() == fg.cpu().reshape(B * K, HW).sum(1).int()).all()


@pytest.mark.parametrize('K', [33, 64])
def test_qt_aux_mask_forms_agree(K_, K):
    """The streaming form (K > 32) forms every value like the register form: each object's logits are the same bits as
    in a 32-object call, and objects whose probability rounds to zero (1 - p == 1, log-odds at the clamp floor) leave
    the other objects' foreground decisions bit-identical to the 32-object call."""
    B, HW = 2, 1620
    pix, w, b = _aux_inputs(B, K, HW, 70 + K)
    pix = pix.view(B, K, 256, HW)
    pix[:, 32:] = 1000.0 * (w < 0).float().view(1, 1, 256, 1)     # relu(x) . w ~ -1e4: sigmoid underflows to 0
    pix32 = pix[:, :32].contiguous().view(B * 32, 256, HW).cuda()
    l32, f32, c32 = K_.qt_aux_mask(pix32, w.cuda(), b.cuda(), B, 32)
    lk, fk, ck_ = K_.qt_aux_mask(pix.reshape(B * K, 256, HW).cuda(), w.cuda(), b.cuda(), B, K)
    assert torch.equal(lk[:, :32], l32)
    assert torch.equal(fk[:, :32], f32)
    assert not fk[:, 32:].any()
    assert torch.equal(ck_.view(B, K)[:, :32], c32.view(B, 32))


# ---------------------------------------------------------------------------------------------
# end to end
# ---------------------------------------------------------------------------------------------
FIFO = dict(mem_every=3, max_mem_frames=4)
LONG = dict(mem_every=1, use_long_term=True, long_term=dict(max_mem_frames=4, min_mem_frames=2, num_prototypes=64,
                                                             max_num_tokens=100, buffer_tokens=20))


def _teacher_forced(cfg, frames, inputs, deletes=None, check=None):
    """tests/test_gpu_e2e.py::test_teacher_forced_vs_cpu_oracle's comparison: every frame starts from the CPU oracle's
    exact state, one step runs on each side, and the segmentation logits must agree within 1e-3.  Near-tied top-k sets
    (SelectionReconciler) and near-tied foreground pixels of the aux masks (ForegroundReconciler: with many objects two
    log-odds within rounding of each other are more frequent) are arbitrated against the oracle's own margins.
    `inputs` {frame: (mask, objects)}, `deletes` {frame: objects deleted before that frame's step}."""
    import cutie_b200.kernels as K_
    from cutie_b200.inference.inference_core import InferenceCore
    from oracle.cpu_core import OracleCore
    from tests.state_sync import ForegroundReconciler, SelectionReconciler, load_state_from_oracle
    from tests.test_gpu_e2e import _net
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    proc, oracle = InferenceCore(_net(cfg), cfg=cfg), OracleCore(_net(cfg, cuda=False), cfg)
    rec = SelectionReconciler(cfg.top_k)
    real_topk, real_aux = K_.affinity_topk, K_.qt_aux_mask
    # Both sides read the buckets in the same order: one top-k call and the same number of aux-mask calls per bucket.
    fgr, gpu_idx, gpu_fg, read = None, [], [], {'reads': 0, 'bucket': -1}

    def spy(*a, **kw):
        r = real_topk(*a, **kw)
        gpu_idx.append(r[0])
        read['reads'] += 1
        return r

    def select(*a):
        rec.gpu_idx = gpu_idx.pop(0)
        return rec(*a)

    def spy_aux(*a, **kw):
        r = real_aux(*a, **kw)
        gpu_fg.append(r[1].clone())
        return r

    def fg_hook(stage, lg, fg):
        if stage == 0:
            read['bucket'] += 1
        n = len(gpu_fg) // max(read['reads'], 1)
        fgr.gpu_fg = gpu_fg[read['bucket'] * n:(read['bucket'] + 1) * n]
        return fgr(stage, lg, fg)
    oracle.selection_hook, oracle.fg_hook = select, fg_hook

    worst = 0.0
    K_.affinity_topk, K_.qt_aux_mask = spy, spy_aux
    try:
        with torch.inference_mode():
            for ti in range(frames.shape[0]):
                load_state_from_oracle(proc, oracle, 'cuda')
                fgr = ForegroundReconciler()
                gpu_idx.clear()
                gpu_fg.clear()
                read.update(reads=0, bucket=-1)
                for o in (deletes or {}).get(ti, ()):
                    proc.delete_objects([o])
                    oracle.delete_objects([o])
                if ti in inputs:
                    m, objs = inputs[ti]
                    pg = proc.step(frames[ti].cuda(), m.cuda(), objects=objs)
                    pc = oracle.step(frames[ti], m, objects=objs)
                else:
                    pg, pc = proc.step(frames[ti].cuda()), oracle.step(frames[ti])
                if ti > 0:
                    err = float((proc.last_logits.cpu() - oracle.last_logits).abs().max())
                    worst = max(worst, err)
                    assert err < 1e-3, (ti, err)
                assert float((pg.cpu() - pc).abs().max()) < 1e-3, ti
                if check is not None:
                    check(ti, proc, oracle)
    finally:
        K_.affinity_topk, K_.qt_aux_mask = real_topk, real_aux
    assert rec.flips <= 0.02 * max(rec.queries, 1) + 2
    return worst


@pytest.mark.parametrize('over,K,T', [(FIFO, 20, 8), (LONG, 40, 8)])
def test_teacher_forced_many_objects_vs_cpu_oracle(over, K, T, monkeypatch):
    """240x432 with 20 (FIFO) and 40 (long-term) objects.  The long-term clip consolidates twice and removes obsolete
    prototypes once (counted here); memory sizes, keys, values and prototype shrinkage are compared with the oracle on
    every frame."""
    import cutie_b200.kernels as K_
    from cutie_b200.config import default_config
    from cutie_b200.inference.memory_bank import KeyValueMemoryStore
    from oracle.synth import synthetic_video
    calls = {'consolidate': 0, 'obsolete': 0}
    real_cons, real_obs = K_.consolidate, KeyValueMemoryStore.remove_obsolete_features

    def cons(*a, **kw):
        calls['consolidate'] += 1
        assert len(a[3]) == K
        return real_cons(*a, **kw)

    def obs(self, *a, **kw):
        calls['obsolete'] += 1
        return real_obs(self, *a, **kw)

    monkeypatch.setattr(K_, 'consolidate', cons)
    monkeypatch.setattr(KeyValueMemoryStore, 'remove_obsolete_features', obs)
    cfg = default_config(**over)
    frames, mask = synthetic_video(T, 240, 432, K, seed=5)

    def check(ti, proc, oracle):
        m = proc.memory
        assert m.work_mem.size(0) == oracle.work.size(0)
        assert torch.allclose(m.work_mem.key[0].cpu(), oracle.work.k[0], atol=1e-4)
        assert torch.allclose(m.work_mem.value[K].cpu(), oracle.work.v[K], rtol=1e-3, atol=2e-3)
        if cfg.use_long_term:
            assert m.long_mem.size(0) == oracle.long.size(0)
            if m.long_mem.size(0):
                assert torch.allclose(m.long_mem.shrinkage[0].cpu().sort(-1)[0], oracle.long.s[0].sort(-1)[0],
                                      rtol=1e-3, atol=1e-3)

    assert _teacher_forced(cfg, frames, {0: (mask, list(range(1, K + 1)))}, check=check) < 1e-3
    if cfg.use_long_term:
        assert calls['consolidate'] >= 2 and calls['obsolete'] >= 1, calls


def test_cuda_graph_many_objects_matches_eager():
    """The K = 20 clip free-running with use_cuda_graphs=True vs the eager path, with the bars
    tests/test_gpu_e2e.py::test_cuda_graph_frame_path_matches_eager sets for 3 objects."""
    from cutie_b200.config import default_config
    from cutie_b200.inference.inference_core import InferenceCore
    from oracle.synth import synthetic_video
    from tests.test_gpu_e2e import _net, _sizes
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = False
    K, T = 20, 8
    cfg = default_config(**FIFO)
    net = _net(cfg)
    eager, graphed = InferenceCore(net, cfg=cfg), InferenceCore(net, cfg=cfg, use_cuda_graphs=True)
    frames, mask = synthetic_video(T, 240, 432, K, seed=5)
    objs = list(range(1, K + 1))
    with torch.inference_mode():
        for ti in range(T):
            a = frames[ti].cuda()
            if ti == 0:
                pe = eager.step(a, mask.cuda(), objects=objs)
                pg = graphed.step(a, mask.cuda(), objects=objs)
            else:
                pe, pg = eager.step(a), graphed.step(a)
                assert float((eager.last_logits - graphed.last_logits).abs().max()) < 2e-4, ti
            assert float((pe - pg).abs().max()) < 1e-4, ti
            assert _sizes(eager) == _sizes(graphed)
    assert graphed._graphs is not None and len(graphed._graphs._seg) >= 1


def test_second_bucket_and_delete_many_objects():
    """20 objects on frame 0 (one bucket), 5 more on frame 3 (a second bucket), then one object of each bucket is
    deleted; teacher-forced against the CPU oracle on every frame."""
    from cutie_b200.config import default_config
    from oracle.synth import synthetic_video
    cfg = default_config(mem_every=2, max_mem_frames=3)
    frames, mask = synthetic_video(8, 240, 432, 20, seed=9)
    extra = torch.zeros_like(mask)
    for j in range(5):
        extra[170:220, 20 + 80 * j:70 + 80 * j] = 21 + j

    def check(ti, proc, oracle):
        buckets = proc.memory.work_mem.buckets
        assert sorted(len(v) for v in buckets.values()) == sorted(len(v) for v in oracle.work.buckets.values())
        if 3 <= ti:
            assert len(buckets) == 2
        assert sum(len(v) for v in buckets.values()) == (20 if ti < 3 else 25 if ti < 6 else 23)

    worst = _teacher_forced(cfg, frames, {0: (mask, list(range(1, 21))), 3: (extra, list(range(21, 26)))},
                            deletes={6: (2, 22)}, check=check)
    assert worst < 1e-3


def test_free_running_many_objects_vs_reference_fixture():
    """20 objects, FIFO memory, 96x160, free-running against the unmodified reference's logits and final probabilities
    (kept at every `logits_stride`-th row and column)."""
    from cutie_b200.config import default_config
    from cutie_b200.inference.inference_core import InferenceCore
    from oracle.synth import synthetic_video
    from tests.test_gpu_e2e import _net, _sizes
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = np.load(os.path.join(GOLDEN, 'e2e_many_objects.npz'))
    T, H, W, K, st = int(g['T']), int(g['H']), int(g['W']), int(g['K']), int(g['logits_stride'])
    cfg = default_config(mem_every=2, max_mem_frames=3)
    proc = InferenceCore(_net(cfg), cfg=cfg)
    frames, mask = synthetic_video(T, H, W, K, seed=3)
    li, worst = 0, 0.0
    with torch.inference_mode():
        for ti in range(T):
            if ti == 0:
                prob = proc.step(frames[0].cuda(), mask.cuda(), objects=list(range(1, K + 1)))
            else:
                prob = proc.step(frames[ti].cuda())
            assert _sizes(proc) == [int(x) for x in g['sizes'][ti] if x >= 0]
            if ti > 0:
                got = proc.last_logits.cpu().numpy()[:, :, ::st, ::st]
                worst = max(worst, float(np.abs(got - g['logits'][li:li + 1]).max()))
                li += 1
    assert worst < 1e-3, worst
    assert float((prob.cpu()[:, ::st, ::st] - torch.from_numpy(g['final_prob'])).abs().max()) < 1e-3
