"""Working / long-term / sensory / object memory and THE READOUT (SURVEY.md section 8 rows a3, a17, a18).

Public surface and semantics follow cutie/inference/memory_manager.py:14-383; the execution plan does not:

  read()         one fused affinity pass per bucket (similarity -> exact top-k -> softmax, never
                 materialising the [N, HW] matrix the reference builds four times, memory_utils.py:28-66),
                 then a sparse k-row gather readout instead of a dense [K*CV, N] x [N, HW] GEMM
                 (memory_manager.py:77-88); no per-frame torch.stack of the value bank (:90-110).
  add_memory()   new tokens are transposed straight into preallocated token-major arena slots; FIFO and
                 consolidation evictions advance a ring head.
  consolidation  prototype rows are gathered and potentiated by kernels writing directly into the
                 long-term arena.
"""
import logging
from typing import Dict, List, Optional

import torch

from cutie_b200 import kernels as K_
from cutie_b200.inference.memory_bank import KeyValueMemoryStore
from cutie_b200.inference.object_manager import ObjectManager

log = logging.getLogger()


def complete_seeds(seeds: torch.Tensor, top_k: int, n_total: int, frame_tokens: int, width: int = 0) -> torch.Tensor:
    """Threshold seeds [B, Q, kpad] in which the winners the ring has dropped since the last read are -1: those slots take
    tokens of the NEWEST memory frame (the last `frame_tokens` tokens of the bank) -- the j-th dropped slot of query q the
    token of the j-th nearest pixel to q's own position in that frame (`width` = feature-map width; 0 = raster neighbours),
    where a temporally coherent video has its best new matches, so the seed bound stays close to the true k-th energy.
    A drop only ever follows an append, so the newest frame was not in the bank at the last read: its tokens cannot
    coincide with a surviving winner, and distinct slots get distinct tokens -- the list stays k DISTINCT valid tokens,
    which is all the threshold needs (results never depend on seeds).  Padding slots (>= top_k) stay -1."""
    B, Q, kpad = seeds.shape
    if frame_tokens < 1 or n_total < frame_tokens or 2 * top_k > frame_tokens:
        return seeds
    dev = seeds.device
    offs = _neighbour_offsets(top_k, width, frame_tokens, dev).to(seeds.dtype)         # [top_k], distinct mod frame_tokens
    q = torch.arange(Q, device=dev, dtype=seeds.dtype).view(1, Q, 1)
    s = torch.arange(kpad, device=dev, dtype=seeds.dtype).view(1, 1, kpad)
    missing = (seeds < 0) & (s < top_k)
    rank = (torch.cumsum(missing.to(torch.int64), dim=2) - 1).clamp_(0, top_k - 1)    # j of the j-th dropped slot
    fill = (n_total - frame_tokens) + torch.remainder(q + offs[rank], frame_tokens)
    return torch.where(missing, fill.to(seeds.dtype), seeds)


_NEIGHBOURS = {}


def _neighbour_offsets(n: int, width: int, frame_tokens: int, device) -> torch.Tensor:
    """Linear offsets of the n nearest pixels (the pixel itself first) on a feature map `width` wide, nearest first --
    DISTINCT modulo frame_tokens (k seeds must be k different tokens: a duplicate would void the bound); on maps too small
    for that, or without a width, the raster neighbours 0, +1, -1, +2, ... (distinct modulo any frame of > 2 n tokens)."""
    key = (n, width, frame_tokens, str(device))
    t = _NEIGHBOURS.get(key)
    if t is None:
        lin = None
        if width > 0:
            r = 1
            while (2 * r + 1) ** 2 < n:
                r += 1
            cand = sorted(((dy * dy + dx * dx, abs(dy), dy, dx) for dy in range(-r, r + 1) for dx in range(-r, r + 1)))
            lin = [dy * width + dx for _, _, dy, dx in cand[:n]]
            if len({o % frame_tokens for o in lin}) < n:
                lin = None
        if lin is None:
            lin = [(j + 1) // 2 * (1 if j % 2 else -1) for j in range(n)]
            assert len({o % frame_tokens for o in lin}) == n
        t = _NEIGHBOURS[key] = torch.tensor(lin, dtype=torch.int64, device=device)
    return t


class MemoryManager:
    def __init__(self, cfg, object_manager: ObjectManager, *, shard_group=None, object_shards=None):
        """shard_group (a torch.distributed process group, or None): key-shard THIS stream's memory over the group's
        ranks (SURVEY.md 8(e).2).  Every rank runs the same frames through the same model; each stores the slice
        shard_bounds(HW, world, rank) of every memory frame's tokens and the read exchanges top-k candidates
        (all_gather) and partial readouts (all_reduce) -- cutie_b200/inference/sharded.py.  With use_long_term the
        long-term store is sharded too: prototypes are chosen by a global usage ranking, potentiated shard-wise (all_gather
        of the per-shard affinity maxima and exp-sums) and dealt to the ranks in contiguous blocks of that ranking.

        object_shards (an object_shards.ObjectShards, or None): keys, shrinkage, selections, top-k, usage and long-term
        maintenance are kept for every object on every rank (the same decisions everywhere); value arrays, sensory
        state and object summaries only for the objects this rank owns.  read() then returns this rank's objects."""
        self.object_manager = object_manager
        self.object_shards = object_shards
        self.shard_group = shard_group
        self.shard_world, self.shard_rank = 1, 0
        if shard_group is not None:
            import torch.distributed as dist
            self.shard_world, self.shard_rank = dist.get_world_size(shard_group), dist.get_rank(shard_group)
            if cfg.use_long_term and cfg.long_term.num_prototypes < self.shard_world:
                raise ValueError(f'{cfg.long_term.num_prototypes} prototypes per consolidation cannot be dealt to '
                                 f'{self.shard_world} ranks (every rank stores at least one)')
        self.sensory_dim = cfg.model.sensory_dim
        self.top_k = cfg.top_k
        self.chunk_size = cfg.chunk_size
        self.save_aux = cfg.save_aux
        self.use_long_term = cfg.use_long_term
        self.count_long_term_usage = cfg.long_term.count_usage
        self._read_sizes(cfg)

        self.CK = self.CV = None
        self.H = self.W = None
        self.sensory: Dict[int, torch.Tensor] = {}      # obj -> [B, C, h, w]
        self.obj_v: Dict[int, torch.Tensor] = {}        # obj -> [B, Q, E+1] running sums | area
        self.work_mem = KeyValueMemoryStore(save_selection=self.use_long_term, save_usage=self.use_long_term,
                                            ring=True)
        if self.use_long_term:
            self.long_mem = KeyValueMemoryStore(save_usage=self.count_long_term_usage, ring=False,
                                                key_centres=self.work_mem.key_centres)
        if object_shards is not None:
            owns = lambda o: object_shards.owner[o] == object_shards.rank          # noqa: E731
            self.work_mem.keeps_values = owns
            if self.use_long_term:
                self.long_mem.keeps_values = owns
        self.config_stale = True
        self.engaged = False
        self.aux = None
        self._prev_topk = {}           # bucket -> (idx of the last read, layout tag): threshold seeds of the next read
        # key-sharded long-term memory: bucket -> long-term tokens held by EVERY rank (a deterministic function of the
        # consolidations / removals so far: no collective is needed to place a rank's tokens in the global index space)
        self._long_counts: Dict[int, List[int]] = {}

    def _read_sizes(self, cfg):
        # the first frame lives in permanent memory and is not counted (memory_manager.py:27-38)
        if self.use_long_term:
            lt = cfg.long_term
            self.max_mem_frames = lt.max_mem_frames - 1
            self.min_mem_frames = lt.min_mem_frames - 1
            self.num_prototypes = lt.num_prototypes
            self.max_long_tokens = lt.max_num_tokens
            self.buffer_tokens = lt.buffer_tokens
        else:
            self.max_mem_frames = cfg.max_mem_frames - 1

    def update_config(self, cfg) -> None:
        self.config_stale = True
        self.top_k = cfg['top_k']
        assert self.use_long_term == cfg.use_long_term, 'cannot update this'
        assert self.count_long_term_usage == cfg.long_term.count_usage, 'cannot update this'
        self._read_sizes(cfg)

    # -- helpers -----------------------------------------------------------------------------
    def local_ids(self, obj_ids: List[int]) -> List[int]:
        """The objects of `obj_ids` whose values / sensory / summaries this manager holds (object sharding: the ones
        this rank owns), in the order of `obj_ids`."""
        return list(obj_ids) if self.object_shards is None else self.object_shards.local(obj_ids)

    def _get_mask_by_ids(self, mask: torch.Tensor, obj_ids: List[int]) -> torch.Tensor:
        return mask[:, [self.object_manager.find_tmp_by_id(o) - 1 for o in obj_ids]]

    def _get_sensory_by_ids(self, obj_ids: List[int]) -> torch.Tensor:
        return torch.stack([self.sensory[o] for o in obj_ids], dim=1)

    def _get_object_mem_by_ids(self, obj_ids: List[int]) -> Optional[torch.Tensor]:
        if obj_ids[0] not in self.obj_v:
            return None
        return torch.stack([self.obj_v[o] for o in obj_ids], dim=1)

    def _topk(self, bucket_id: int, qk: torch.Tensor, qe: torch.Tensor):
        """Affinity -> top-k -> softmax (+ usage commits) for one bucket.  Returns gather(objects) -> [B,K,CV,Q]."""
        bs = qk.shape[0]
        if self.shard_group is not None:
            from cutie_b200.inference.sharded import shard_bounds, sharded_gather, sharded_topk
            key_segs = self._segments(bucket_id, [])
            n_local = sum(s.n for s in key_segs)
            long_all = self._long_counts.get(bucket_id, [0] * self.shard_world)
            long_n = long_all[self.shard_rank]
            frames, rem = divmod(n_local - long_n, self.HW)    # self.HW is the LOCAL tokens per frame here
            assert rem == 0 and frames >= 1
            # global index space = the ranks' local banks (long-term | permanent | temporary) one after the other
            per_rank = [long_all[r] + frames * (lambda be: be[1] - be[0])(shard_bounds(self.HW_global, self.shard_world, r))
                        for r in range(self.shard_world)]
            assert per_rank[self.shard_rank] == n_local
            usage_acc = None
            if self.use_long_term:
                usage_acc = torch.zeros(bs, n_local, dtype=torch.int64, device=qk.device)
            idx_l, w_l, _, _ = sharded_topk(key_segs, sum(per_rank[:self.shard_rank]), sum(per_rank), qk, qe, self.top_k,
                                            self.shard_group, usage_acc_local=usage_acc)
            if self.use_long_term:
                self.work_mem.update_bucket_usage(bucket_id, usage_acc, long_n + self.work_mem.perm_size(bucket_id))
                if long_n and self.count_long_term_usage:
                    self.long_mem.update_bucket_usage(bucket_id, usage_acc, 0)
            return lambda objects: sharded_gather(idx_l, w_l, self._segments(bucket_id, objects), self.shard_group)
        long_n = self.long_mem.size(bucket_id) if (self.use_long_term and self.long_mem.engaged(bucket_id)) else 0
        key_segs = self._segments(bucket_id, [])
        usage_acc = None
        if self.use_long_term:
            usage_acc = torch.zeros(bs, sum(s.n for s in key_segs), dtype=torch.int64, device=qk.device)
        seed, tag = self._threshold_seeds(bucket_id, qk)
        idx, wgt, _ = K_.affinity_topk(key_segs, qk, qe, self.top_k, usage_acc=usage_acc, seed_idx=seed)
        if tag is not None:
            self._prev_topk[bucket_id] = (idx,) + tag
        if self.use_long_term:
            # usage of the temporary working tokens; permanent tokens are skipped (kv:157)
            self.work_mem.update_bucket_usage(bucket_id, usage_acc, long_n + self.work_mem.perm_size(bucket_id))
            if long_n and self.count_long_term_usage:
                self.long_mem.update_bucket_usage(bucket_id, usage_acc, 0)
        return lambda objects: K_.readout_gather(idx, wgt, self._segments(bucket_id, objects))

    def _threshold_seeds(self, bucket_id: int, qk: torch.Tensor):
        """The previous read's winners of this bucket, re-indexed for what the ring dropped since, as threshold seeds for
        the candidate filter (kernels.affinity_topk(seed_idx=...)): in a temporally coherent video the k tokens that won
        for a pixel on the last frame are still (nearly) the k best, so the largest of their exact energies is a far
        tighter bound than a sampled one.  Exactness never depends on them.  FIFO working memory only (long-term
        consolidation re-orders tokens): returns (seed or None, tag to store with this read's result or None)."""
        if self.use_long_term:
            return None, None
        bk = self.work_mem._b[bucket_id]
        tag = (bk.perm.count, bk.perm.generation, bk.temp.generation, bk.temp.total_dropped, tuple(qk.shape))
        prev = self._prev_topk.get(bucket_id)
        if prev is None:
            return None, tag
        idx, P, gp, gt, dropped0, shape = prev
        if (P, gp, gt, shape) != (tag[0], tag[1], tag[2], tag[4]):
            return None, tag
        d = bk.temp.total_dropped - dropped0
        if d == 0:
            return idx, tag
        moved = idx - d                                  # temporary tokens slid towards the permanent prefix by d
        seeds = torch.where(idx < P, idx, torch.where(moved >= P, moved, torch.full_like(idx, -1)))
        return complete_seeds(seeds, self.top_k, self.work_mem.size(bucket_id), self.HW, self.W or 0), tag

    def _segments(self, bucket_id: int, obj_ids: List[int]):
        segs = []
        if self.use_long_term and self.long_mem.engaged(bucket_id):
            segs += self.long_mem.segments(bucket_id, obj_ids)
        return segs + self.work_mem.segments(bucket_id, obj_ids)

    # -- the readout ---------------------------------------------------------------------------
    def read(self, pix_feat: torch.Tensor, query_key: torch.Tensor, selection: torch.Tensor,
             last_mask: torch.Tensor, network) -> Dict[int, torch.Tensor]:
        """pix_feat [B,C,h,w]; query_key/selection [B,CK,h,w]; last_mask [B,K,H,W] -> {obj: [B,CV,h,w]}."""
        h, w = pix_feat.shape[-2:]
        bs = pix_feat.shape[0]
        assert query_key.shape[0] == bs
        assert selection.shape[0] == bs
        assert last_mask.shape[0] == bs
        qk = query_key.flatten(2).contiguous()
        qe = selection.flatten(2).contiguous()

        out: Dict[int, torch.Tensor] = {}
        for bucket_id, bucket in self.work_mem.buckets.items():
            gather = self._topk(bucket_id, qk, qe)

            if self.object_shards is not None:       # chunk_size < 1, save_aux off (InferenceCore checks)
                grp = self.object_shards.group_of(bucket)
                objects = grp.local_ids
                if not objects:
                    if getattr(network, 'object_transformer_enabled', True):
                        network.object_transformer.exchange_without_objects(grp, bs, h * w, pix_feat.device)
                    continue
                visual = gather(objects).view(bs, len(objects), self.CV, h, w)
                pixel_readout = network.pixel_fusion(pix_feat, visual, self._get_sensory_by_ids(objects),
                                                     self._get_mask_by_ids(last_mask, bucket), objects=grp)
                obj_mem = self._get_object_mem_by_ids(objects)
                obj_mem = obj_mem.unsqueeze(2) if obj_mem is not None else None
                readout_memory, _ = network.readout_query(pixel_readout, obj_mem, objects=grp)
                for i, o in enumerate(objects):
                    out[o] = readout_memory[:, i]
                continue

            if self.chunk_size < 1:
                chunks = [bucket]
            else:
                chunks = [bucket[i:i + self.chunk_size] for i in range(0, len(bucket), self.chunk_size)]
            for objects in chunks:
                this_sensory = self._get_sensory_by_ids(objects)
                this_last_mask = self._get_mask_by_ids(last_mask, objects)
                visual = gather(objects).view(bs, len(objects), self.CV, h, w)
                pixel_readout = network.pixel_fusion(pix_feat, visual, this_sensory, this_last_mask)
                obj_mem = self._get_object_mem_by_ids(objects)
                obj_mem = obj_mem.unsqueeze(2) if obj_mem is not None else None
                readout_memory, aux_features = network.readout_query(pixel_readout, obj_mem)
                for i, o in enumerate(objects):
                    out[o] = readout_memory[:, i]
                if self.save_aux:
                    self.aux = {
                        'sensory': this_sensory,
                        'pixel_readout': pixel_readout,
                        'q_logits': aux_features['logits'] if aux_features else None,
                        'q_weights': aux_features['q_weights'] if aux_features else None,
                        'p_weights': aux_features['p_weights'] if aux_features else None,
                        'attn_mask': (network.object_transformer.attn_mask_from_fg(aux_features['fg_map']).float()
                                      if aux_features else None),
                    }
        return out

    def read_visual(self, query_key: torch.Tensor, selection: torch.Tensor, obj_ids: List[int]) -> torch.Tensor:
        """The memory half of read() for the single-bucket, un-chunked case: fused affinity + sparse value gather
        (+ usage commits) -> visual readout [B, K, CV, h, w].  Used by the CUDA-graph frame path, which runs the
        fusion / object-transformer / decoder half as one graph replay."""
        h, w = query_key.shape[-2:]
        bs = query_key.shape[0]
        qk = query_key.flatten(2).contiguous()
        qe = selection.flatten(2).contiguous()
        (bucket_id, bucket), = self.work_mem.buckets.items()
        assert list(bucket) == list(obj_ids)
        return self._topk(bucket_id, qk, qe)(bucket).view(bs, len(bucket), self.CV, h, w)

    # -- insertion -----------------------------------------------------------------------------
    def add_memory(self, key: torch.Tensor, shrinkage: torch.Tensor, msk_value: torch.Tensor,
                   obj_value: Optional[torch.Tensor], objects: List[int],
                   selection: Optional[torch.Tensor] = None, *, as_permanent='no') -> None:
        """key [B,CK,h,w]; shrinkage [B,1,h,w]; msk_value [B,K,CV,h,w]; obj_value [B,K,Q,E+1].
        Object sharding: `objects` are all objects of the frame, msk_value / obj_value hold local_ids(objects)."""
        bs = key.shape[0]
        assert shrinkage.shape[0] == bs
        assert msk_value.shape[0] == bs
        assert obj_value is None or obj_value.shape[0] == bs

        self.engaged = True
        if self.H is None or self.config_stale:
            self.config_stale = False
            self.H, self.W = key.shape[-2:]
            self.HW = self.HW_global = self.H * self.W
            if self.shard_group is not None:              # sizes below are in LOCAL tokens (this rank's slice)
                from cutie_b200.inference.sharded import shard_bounds
                self.shard_begin, self.shard_end = shard_bounds(self.HW_global, self.shard_world, self.shard_rank)
                self.HW = self.shard_end - self.shard_begin
                if self.HW < 1:
                    raise ValueError(f'{self.HW_global} tokens per frame cannot be sharded over {self.shard_world} ranks')
            self.max_work_tokens = self.max_mem_frames * self.HW
            if self.use_long_term:
                self.min_work_tokens = self.min_mem_frames * self.HW
                self.long_mem.set_capacity_hint(temp_tokens=self.max_long_tokens + self.num_prototypes)
            self.work_mem.set_capacity_hint(temp_tokens=self.max_work_tokens + self.HW, perm_tokens=self.HW)

        key = key.flatten(2)
        shrinkage = shrinkage.flatten(2)
        self.CK = key.shape[1]
        msk_value = msk_value.flatten(3)
        self.CV = msk_value.shape[2]
        if selection is not None:
            selection = selection.flatten(2)
        if self.shard_group is not None:                  # keep this rank's slice of the frame's tokens
            sl = slice(self.shard_begin, self.shard_end)
            key, shrinkage, msk_value = key[:, :, sl], shrinkage[:, :, sl], msk_value[:, :, :, sl]
            selection = selection[:, :, sl] if selection is not None else None

        local = self.local_ids(objects)
        if obj_value is not None:                       # streaming sums (memory_manager.py:252-271)
            for i, obj in enumerate(local):
                new = obj_value[:, i].contiguous()
                if obj in self.obj_v:
                    K_.obj_summary_accumulate(self.obj_v[obj], new)
                else:
                    self.obj_v[obj] = new.clone()

        values = {obj: msk_value[:, i] for i, obj in enumerate(local)}
        self.work_mem.add(key, values, shrinkage, selection=selection, as_permanent=as_permanent,
                          objects=objects if self.object_shards is not None else None)

        for bucket_id in self.work_mem.buckets.keys():
            if self.use_long_term:
                if self.work_mem.non_perm_size(bucket_id) >= self.max_work_tokens:
                    # long-term sizes are GLOBAL token counts (sharded: the sum over the ranks; every rank takes the
                    # same branch, the branches contain collectives)
                    long_size = (sum(self._long_counts.get(bucket_id, [0])) if self.shard_group is not None
                                 else self.long_mem.non_perm_size(bucket_id))
                    if long_size >= (self.max_long_tokens - self.num_prototypes):
                        keep = self.max_long_tokens - self.num_prototypes - self.buffer_tokens
                        if self.shard_group is not None:
                            self._remove_obsolete_sharded(bucket_id, keep)
                        else:
                            self.long_mem.remove_obsolete_features(bucket_id, keep)
                    self.compress_features(bucket_id)
            else:
                self.work_mem.remove_old_memory(bucket_id, self.max_work_tokens)

    def purge_except(self, obj_keep_idx: List[int]) -> None:
        """memory_manager.py:298-307 -- including its quirk: obj_v entries of purged objects are kept."""
        self._prev_topk.clear()
        self.work_mem.purge_except(obj_keep_idx)
        if self.use_long_term and self.long_mem.engaged():
            self.long_mem.purge_except(obj_keep_idx)
            self._long_counts = {b: c for b, c in self._long_counts.items() if self.long_mem.engaged(b)}
        self.sensory = {k: v for k, v in self.sensory.items() if k in obj_keep_idx}
        if not self.work_mem.engaged():
            self.engaged = False

    # -- long-term consolidation (memory_manager.py:309-358) -------------------------------------
    def compress_features(self, bucket_id: int) -> None:
        n_temp = self.work_mem.non_perm_size(bucket_id)
        n_cand = n_temp - self.min_work_tokens
        self.consolidation(bucket_id, n_cand)
        self.work_mem.sieve_by_range(bucket_id, 0, -self.min_work_tokens, min_size=self.min_work_tokens)

    def consolidation(self, bucket_id: int, n_cand: int) -> None:
        """Candidates = the n_cand oldest temporary working tokens.  Prototypes = the num_prototypes most
        used candidates (:339); their values/shrinkage are the dense-softmax readout of all candidates
        (:348-356).  Results are written straight into new long-term arena slots."""
        if self.shard_group is not None:
            return self._consolidation_sharded(bucket_id, n_cand)
        objs = self.work_mem.buckets[bucket_id]
        vobjs = self.local_ids(objs)
        arena, runs = self.work_mem.temp_runs(bucket_id, 0, n_cand)
        bs = arena.B
        dev = arena.device
        use = torch.cat([arena.view('use', r) for r in runs], 1)
        life = torch.cat([arena.view('life', r) for r in runs], 1)
        proto_idx = torch.topk(use / life, k=self.num_prototypes, dim=-1, sorted=True)[1]     # [B, P]
        P = self.num_prototypes
        slots = self.long_mem.slots_for_add(objs, P, bs, self.CK, self.CV, dev, supposed_bucket_id=bucket_id)
        (_, larena, lruns, _), = slots
        (lrun,) = lruns
        K_.bank_gather([arena.view('key', r) for r in runs], proto_idx, larena.view('key', lrun))
        proto_sel = torch.empty(bs, P, self.CK, dtype=torch.float32, device=dev)
        K_.bank_gather([arena.view('sel', r) for r in runs], proto_idx, proto_sel)
        cand = self.work_mem.segments(bucket_id, vobjs, perm=False, temp_start=0, temp_len=n_cand)
        K_.consolidate(cand, larena.view('key', lrun), proto_sel,
                       [larena.view(('val', o), lrun) for o in vobjs], larena.view('shr', lrun))

    # -- the same, key-sharded (cutie_b200/inference/sharded.py) ---------------------------------------
    def _consolidation_sharded(self, bucket_id: int, n_cand: int) -> None:
        """consolidation() with the candidates spread over the ranks (n_cand = this rank's share of them).  Prototypes =
        the global top-P of usage (select_top); their keys / selections are fetched from the owning ranks; every rank
        potentiates against ITS candidates (cutie_consolidate_partial) and the shards' results are combined through an
        all_gather of the per-shard affinity maxima and exp-sums (combine_partial_softmax).  Prototype j of the global
        ranking is stored by the rank whose block shard_bounds(P, world, rank) holds j."""
        from cutie_b200.inference import sharded as S
        g, world, rank = self.shard_group, self.shard_world, self.shard_rank
        objs = self.work_mem.buckets[bucket_id]
        arena, runs = self.work_mem.temp_runs(bucket_id, 0, n_cand)
        bs, dev, P, CK, CV = arena.B, arena.device, self.num_prototypes, self.CK, self.CV
        use = torch.cat([arena.view('use', r) for r in runs], 1)
        life = torch.cat([arena.view('life', r) for r in runs], 1)
        src_rank, src_idx = S.select_top(use / life, P, g)
        proto_key = S.fetch_rows([arena.view('key', r) for r in runs], src_rank, src_idx, g)
        proto_sel = S.fetch_rows([arena.view('sel', r) for r in runs], src_rank, src_idx, g)
        cand = self.work_mem.segments(bucket_id, objs, perm=False, temp_start=0, temp_len=n_cand)
        vals = [torch.empty(bs, P, CV, dtype=torch.float32, device=dev) for _ in objs]
        shr = torch.empty(bs, P, dtype=torch.float32, device=dev)
        mx, se = torch.empty(bs, P, device=dev), torch.empty(bs, P, device=dev)
        K_.consolidate(cand, proto_key, proto_sel, vals, shr, stats=(mx, se))
        full = S.combine_partial_softmax(torch.cat(vals + [shr.unsqueeze(-1)], dim=-1), mx, se, g)
        lo, hi = S.shard_bounds(P, world, rank)
        (_, larena, lruns, _), = self.long_mem.slots_for_add(objs, hi - lo, bs, CK, CV, dev, supposed_bucket_id=bucket_id)
        (lrun,) = lruns
        larena.view('key', lrun).copy_(proto_key[:, lo:hi])
        for i, o in enumerate(objs):
            larena.view(('val', o), lrun).copy_(full[:, lo:hi, i * CV:(i + 1) * CV])
        larena.view('shr', lrun).copy_(full[:, lo:hi, -1])
        counts = self._long_counts.setdefault(bucket_id, [0] * world)
        for r in range(world):
            b, e = S.shard_bounds(P, world, r)
            counts[r] += e - b
        assert counts[rank] == self.long_mem.non_perm_size(bucket_id)

    def _remove_obsolete_sharded(self, bucket_id: int, max_size: int) -> None:
        """KeyValueMemoryStore.remove_obsolete_features (kv_memory_store.py:209-242) over the ranks: the max_size most used
        long-term tokens of ALL ranks survive, in descending-usage order, and rank r keeps block
        shard_bounds(max_size, world, r) of that ranking (so every rank and every batch entry holds the same count)."""
        from cutie_b200.inference import sharded as S
        g, world, rank = self.shard_group, self.shard_world, self.shard_rank
        src_rank, src_idx = S.select_top(self.long_mem.get_usage(bucket_id), max_size, g)
        lo, hi = S.shard_bounds(max_size, world, rank)
        arena, runs = self.long_mem.temp_runs(bucket_id)
        fresh = {}
        for name, width in arena.widths.items():
            rows = [arena.view(name, r) if width else arena.view(name, r).unsqueeze(-1) for r in runs]
            got = S.fetch_rows(rows, src_rank, src_idx, g)[:, lo:hi]
            fresh[name] = got if width else got.squeeze(-1)
        self.long_mem.replace_temp_rows(bucket_id, fresh)
        self._long_counts[bucket_id] = [(lambda be: be[1] - be[0])(S.shard_bounds(max_size, world, r)) for r in range(world)]

    # -- sensory memory ------------------------------------------------------------------------------
    def initialize_sensory_if_needed(self, sample_key: torch.Tensor, ids: List[int]):
        for obj in ids:
            if obj not in self.sensory:
                bs, _, h, w = sample_key.shape
                self.sensory[obj] = torch.zeros((bs, self.sensory_dim, h, w), device=sample_key.device)

    def update_sensory(self, sensory: torch.Tensor, ids: List[int]):
        for i, obj in enumerate(ids):
            self.sensory[obj] = sensory[:, i]

    def get_sensory(self, ids: List[int]):
        return self._get_sensory_by_ids(ids)

    def clear_non_permanent_memory(self):
        self.work_mem.clear_non_permanent_memory()
        if self.use_long_term:
            self.long_mem.clear_non_permanent_memory()
            self._long_counts.clear()

    def clear_sensory_memory(self):
        self.sensory = {}
