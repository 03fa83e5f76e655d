"""Per-video frame loop (SURVEY.md section 8 rows a1, a2): the drop-in for
cutie.inference.inference_core.InferenceCore (cutie/inference/inference_core.py:18-345).

Same constructor, `step` signature, return value ([1+K, H, W] probabilities) and public attributes
(memory, object_manager, max_internal_size, mem_every, ...), so scripting_demo.py / eval_vos.py /
process_video.py drive it unchanged.  The memory read it calls is the fused-kernel path of
cutie_b200.inference.memory_manager.
"""
import contextlib
import logging
from typing import Iterable, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from cutie_b200 import kernels as K_
from cutie_b200.inference.image_feature_store import ImageFeatureStore
from cutie_b200.inference.memory_manager import MemoryManager
from cutie_b200.inference.object_manager import ObjectManager
from cutie_b200.utils.tensor_utils import aggregate, pad_divide_by, unpad

log = logging.getLogger()


def _graphable(t: torch.Tensor) -> bool:
    """CUDA graphs (and the encoder look-ahead) need CUDA tensors.  A function so that the CPU suite can drive the graph
    path with stand-in graphs (tests/test_graph_path_cpu.py); the product never changes it."""
    return t.is_cuda


def _autocast_state():
    """(enabled, dtype) of CUDA autocast where step() is called.  A function so that the CPU suite can substitute it
    (tests/test_amp_policy_cpu.py: without a GPU torch.autocast('cuda') disables itself); the product never changes it."""
    return torch.is_autocast_enabled('cuda'), torch.get_autocast_dtype('cuda')


class _CudaStreamOps:
    """The torch.cuda calls EncoderLookahead needs (tests substitute a recording fake)."""

    def __init__(self):
        self.side = None

    def _side(self, device):
        if self.side is None or self.side.device != device:
            self.side = torch.cuda.Stream(device=device)
        return self.side

    def side_wait_main(self, device):
        self._side(device).wait_stream(torch.cuda.current_stream())

    def keep_alive_on_side(self, tensor):
        tensor.record_stream(self._side(tensor.device))

    def on_side(self, device):
        return torch.cuda.stream(self._side(device))

    def record_on_side(self, device):
        ev = torch.cuda.Event()
        ev.record(self._side(device))
        return ev

    def main_wait_event(self, ev):
        torch.cuda.current_stream().wait_event(ev)


def _version_of(t: torch.Tensor):
    """In-place modification counter of a tensor, or None for inference tensors (created under torch.inference_mode():
    they carry no counter, so for them a look-ahead hit rests on object identity alone and overwriting an announced
    inference tensor in place before the next step is outside the contract of step(next_image=...))."""
    try:
        return t._version
    except RuntimeError:
        return None


class EncoderLookahead:
    """Which encoder capture slot holds the current frame's features, and the pending look-ahead (if any).

    encode(image, slot) replays the image-encoder graph of `slot` on the CURRENT stream and returns its (graph-static)
    outputs.  Protocol (checked as a happens-before model in tests/test_lookahead_protocol_cpu.py):
      * a look-ahead always writes the slot the current frame does NOT use;
      * before it, the side stream waits for everything enqueued on the main stream so far -- the end of the previous
        step, whose consumers were the last readers of that slot, and whatever made the announced image valid;
      * the main stream waits for the look-ahead's event before it touches either the outputs (hit) or re-encodes
        (miss: wrong frame / tensor announced -- the result is discarded, never used);
      * a look-ahead records the precision mode it was encoded under (`mode`: fp32 or amp); a step in the other mode
        counts it as a miss (the encoder's arithmetic differs between the modes)."""

    def __init__(self, encode, ops=None):
        self.encode = encode
        self.ops = ops or _CudaStreamOps()
        self.slot = 0
        self.pending = None

    def current(self, ti: int, image: torch.Tensor, src_id, mode=None):
        la, self.pending = self.pending, None
        if la is not None:
            self.ops.main_wait_event(la['done'])
            # a hit needs the very memory that was announced, unmodified since: same address / shape / strides, same
            # in-place version counter (views share their base's), and `pending` holds a reference to the announced
            # tensor, so its address cannot have been recycled for another frame in between
            t = la['tensor']
            if (la['ti'] == ti and src_id.data_ptr() == t.data_ptr() and tuple(src_id.shape) == tuple(t.shape)
                    and src_id.stride() == t.stride() and la['version'] == _version_of(src_id)
                    and la['shape'] == tuple(image.shape) and la['mode'] == mode):
                self.slot = la['slot']
                return la['out'], True
        return self.encode(image, self.slot), False

    def ahead(self, ti: int, next_image: torch.Tensor, prepare, mode=None):
        dev = next_image.device
        self.ops.side_wait_main(dev)
        self.ops.keep_alive_on_side(next_image)
        slot = 1 - self.slot
        with self.ops.on_side(dev):
            img = prepare(next_image)
            out = self.encode(img, slot)
            done = self.ops.record_on_side(dev)
        self.pending = dict(ti=ti + 1, slot=slot, tensor=next_image, version=_version_of(next_image),
                            shape=tuple(img.shape), out=out, done=done, mode=mode)


class InferenceCore:
    def __init__(self, network, cfg, *, image_feature_store: ImageFeatureStore = None,
                 use_cuda_graphs: bool = False, memory_shard_group=None, object_shard_group=None):
        """memory_shard_group: split the memory bank's tokens over the group's ranks (MemoryManager).
        object_shard_group: split the video's objects over the group's ranks (object_shards.py): each object's readout,
        fusion, object transformer, decoder and mask encoder run on the rank that owns it.  Every rank of either group
        calls step() with the same arguments and gets the same full result."""
        if object_shard_group is not None:
            if memory_shard_group is not None:
                raise ValueError('object sharding cannot be combined with memory (key) sharding')
            if cfg.chunk_size >= 1:
                raise NotImplementedError('object sharding needs chunk_size < 1: chunks would couple objects per chunk')
            if cfg.save_aux:
                raise NotImplementedError('object sharding does not export auxiliary outputs (save_aux)')
        self.network = network
        self.cfg = cfg
        self.mem_every = cfg.mem_every
        self.chunk_size = cfg.chunk_size
        self.save_aux = cfg.save_aux
        self.max_internal_size = cfg.max_internal_size
        self.flip_aug = cfg.flip_aug

        self.curr_ti = -1
        self.last_mem_ti = 0
        # offsets (in frames since the last memory frame) at which the sensory memory is refreshed
        stagger = cfg.stagger_updates
        if stagger >= self.mem_every:
            self.stagger_ti = set(range(1, self.mem_every + 1))
        else:
            self.stagger_ti = set(np.round(np.linspace(1, self.mem_every, stagger)).astype(int))
        self.object_manager = ObjectManager()
        self.memory_shard_group = memory_shard_group
        self.object_shards = None
        if object_shard_group is not None:
            from cutie_b200.inference.object_shards import ObjectShards
            self.object_shards = ObjectShards(object_shard_group)
        self.memory = MemoryManager(cfg=cfg, object_manager=self.object_manager, shard_group=memory_shard_group,
                                    object_shards=self.object_shards)
        self.image_feature_store = image_feature_store or ImageFeatureStore(self.network)
        self.last_mask = None
        self.last_logits = None      # network.segment(...)[1] of the latest segmented frame (parity hook)
        # replay CUDA graphs for the arena-independent parts of a frame (frame_graphs.py); off = reference-like eager
        self.use_cuda_graphs = use_cuda_graphs
        self._graphs = None
        # encoder look-ahead (step(..., next_image=...)): the next frame's image-encoder graph on a side stream
        self._lookahead = None       # EncoderLookahead, created with the graphs
        self._amp = False            # the current step runs in amp mode (step() under fp16 autocast)

    # -- memory control ------------------------------------------------------------------------
    def _reset_clock(self):
        self.curr_ti = -1
        self.last_mem_ti = 0

    def clear_memory(self):
        self._reset_clock()
        self.memory = MemoryManager(cfg=self.cfg, object_manager=self.object_manager,
                                    shard_group=self.memory_shard_group, object_shards=self.object_shards)

    def clear_non_permanent_memory(self):
        self._reset_clock()
        self.memory.clear_non_permanent_memory()

    def clear_sensory_memory(self):
        self._reset_clock()
        self.memory.clear_sensory_memory()

    def update_config(self, cfg):
        self.mem_every = cfg['mem_every']
        self.memory.update_config(cfg)

    # -- the two halves of a step ------------------------------------------------------------------
    def _add_memory(self, image, pix_feat, prob, key, shrinkage, selection, *, is_deep_update: bool = True,
                    force_permanent: bool = False) -> None:
        """Encode the (predicted or given) masks and append one frame of tokens to the memory."""
        if prob.shape[1] == 0:
            log.warning('Trying to add an empty object mask to memory!')
            return
        ids = self.object_manager.all_obj_ids
        if self.object_shards is not None:
            return self._add_memory_sharded(image, pix_feat, prob, key, shrinkage, selection, ids,
                                            is_deep_update=is_deep_update, force_permanent=force_permanent)
        self.memory.initialize_sensory_if_needed(key, ids)
        graphed = (self.use_cuda_graphs and self._graphs is not None and _graphable(image) and is_deep_update and
                   not self.flip_aug and self.chunk_size < 1 and not self.save_aux and
                   getattr(self.network, 'object_transformer_enabled', True))
        if graphed:
            with K_._call('region:encode_mask_graph', 0):          # bench.py: device time of the whole replay
                msk_value, sensory, obj_value = self._graphs.encode_mask(image, pix_feat, self.memory.get_sensory(ids),
                                                                         prob, amp=self._amp)
            sensory = sensory.clone()          # outlives this frame; value / summaries are consumed by add_memory below
        else:
            msk_value, sensory, obj_value, _ = self.network.encode_mask(
                image, pix_feat, self.memory.get_sensory(ids), prob, deep_update=is_deep_update,
                chunk_size=self.chunk_size, need_weights=self.save_aux)
        self.memory.add_memory(key, shrinkage, msk_value, obj_value, ids, selection=selection,
                               as_permanent='all' if force_permanent else 'first')
        self.last_mem_ti = self.curr_ti
        if is_deep_update:
            self.memory.update_sensory(sensory, ids)

    def _add_memory_sharded(self, image, pix_feat, prob, key, shrinkage, selection, ids, *, is_deep_update: bool,
                            force_permanent: bool) -> None:
        """_add_memory under object sharding: the mask encoder and summarizer run on this rank's objects (the others-mask
        from all of `prob`); keys go to memory on every rank, values only on the owner's."""
        grp = self.object_shards.group_of(ids)
        local = grp.local_ids
        self.memory.initialize_sensory_if_needed(key, local)
        if local:
            msk_value, sensory, obj_value, _ = self.network.encode_mask(
                image, pix_feat, self.memory.get_sensory(local), prob, deep_update=is_deep_update,
                chunk_size=self.chunk_size, objects=grp)
        else:
            msk_value = key.new_empty(key.shape[0], 0, self.network.value_dim, *key.shape[-2:])
            sensory = obj_value = None
        self.memory.add_memory(key, shrinkage, msk_value, obj_value, ids, selection=selection,
                               as_permanent='all' if force_permanent else 'first')
        self.last_mem_ti = self.curr_ti
        if is_deep_update and local:
            self.memory.update_sensory(sensory, local)

    def _segment(self, key, selection, pix_feat, ms_features: Iterable[torch.Tensor],
                 update_sensory: bool = True) -> torch.Tensor:
        """Memory read -> decoder.  Returns [1+K, H, W] probabilities (channel 0 = background)."""
        bs = key.shape[0]
        assert bs == (2 if self.flip_aug else 1)
        if not self.memory.engaged:
            log.warning('Trying to segment without any memory!')
            return torch.zeros((1, key.shape[-2] * 16, key.shape[-1] * 16), device=key.device, dtype=key.dtype)

        ids = self.object_manager.all_obj_ids
        if self._graph_path_ok(key, ids):
            # eager memory read (affinity + sparse gather), then one graph replay for fusion + object transformer +
            # decoder; results live in graph-static buffers, so everything that outlives this frame is cloned
            with K_._call('region:memory_read', 0):
                visual = self.memory.read_visual(key, selection, ids)
            sens_in = self.memory.get_sensory(ids)
            obj_mem = self.memory._get_object_mem_by_ids(ids).unsqueeze(2)
            with K_._call('region:segment_graph', 0):
                last_mask = self.memory._get_mask_by_ids(self.last_mask, ids)     # after delete_objects: live channels only
                sensory, logits, prob = self._graphs.segment(visual, pix_feat, sens_in, last_mask, obj_mem,
                                                             tuple(ms_features), update_sensory, amp=self._amp)
            logits, prob = logits.clone(), prob.clone()
            if update_sensory:
                sensory = sensory.clone()
        elif self.object_shards is not None:
            readout = self.memory.read(pix_feat, key, selection, self.last_mask, self.network)
            grp = self.object_shards.group_of(ids)
            ids = grp.local_ids
            readout = torch.stack([readout[o] for o in ids], dim=1) if ids else None
            sensory, logits, prob = self.network.segment(ms_features, readout,
                                                         self.memory.get_sensory(ids) if ids else None,
                                                         chunk_size=self.chunk_size, update_sensory=update_sensory,
                                                         objects=grp)
            update_sensory = update_sensory and bool(ids)
        else:
            readout = self.memory.read(pix_feat, key, selection, self.last_mask, self.network)
            readout = self.object_manager.realize_dict(readout)
            sensory, logits, prob = self.network.segment(ms_features, readout, self.memory.get_sensory(ids),
                                                         chunk_size=self.chunk_size, update_sensory=update_sensory)
        self.last_logits = logits
        if self.flip_aug:
            prob = (prob[0] + torch.flip(prob[1], dims=[-1])) / 2
        else:
            prob = prob[0]
        if update_sensory:
            self.memory.update_sensory(sensory, ids)
        return prob

    def _graph_path_ok(self, key: torch.Tensor, ids) -> bool:
        if not (self.use_cuda_graphs and _graphable(key)) or self.object_shards is not None:
            return False
        m = self.memory
        if self.flip_aug or self.chunk_size >= 1 or self.save_aux or len(m.work_mem.buckets) != 1:
            return False
        if not getattr(self.network, 'object_transformer_enabled', True) or any(o not in m.obj_v for o in ids):
            return False
        if self._graphs is None:
            from cutie_b200.inference.frame_graphs import FrameGraphs
            self._graphs = FrameGraphs(self.network)
        return list(next(iter(m.work_mem.buckets.values()))) == list(ids)

    def step(self, image: torch.Tensor, mask: Optional[torch.Tensor] = None,
             objects: Optional[List[int]] = None, *, idx_mask: bool = True, end: bool = False,
             delete_buffer: bool = True, force_permanent: bool = False,
             next_image: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One frame.  image [3,H,W] in [0,1]; mask [H,W] ids (idx_mask) or [K,H,W] soft masks or None;
        objects: ids present in `mask`.  With a mask the listed objects are memorised (and any others
        are propagated first); without, the frame is segmented from memory.  Returns [1+K,H,W].

        next_image (extension; CUDA-graph path only): the frame the NEXT call will be given.  Its image encoder -- which
        depends on nothing but the image -- is enqueued on a side stream now and overlaps this frame's memory read,
        object transformer and decoder; the next call picks the result up if it is handed the same tensor.  Results
        are identical with or without it.

        Mixed precision: called under fp16 CUDA autocast (as the reference's scripting_demo.py / eval_vos.py / GUI do),
        the step runs with autocast switched off -- every PyTorch / cuDNN op stays fp32 -- and the model's convolution
        fuser in amp mode: the tensor-core convolutions take their FP16-operand form (fuse.ConvEpilogueFuser 'tc16').
        Inputs and outputs stay fp32.  bf16 autocast raises NotImplementedError."""
        on, dtype = _autocast_state()
        self._amp = bool(on)
        if not on:
            return self._step(image, mask, objects, idx_mask=idx_mask, end=end, delete_buffer=delete_buffer,
                              force_permanent=force_permanent, next_image=next_image)
        if dtype != torch.float16:
            raise NotImplementedError(f'InferenceCore.step under {dtype} autocast: only float16 autocast is supported')
        fuser = getattr(self.network, 'conv_epilogues', None)
        with torch.autocast('cuda', enabled=False), (fuser.amp_mode() if fuser is not None else contextlib.nullcontext()):
            return self._step(image, mask, objects, idx_mask=idx_mask, end=end, delete_buffer=delete_buffer,
                              force_permanent=force_permanent, next_image=next_image)

    def _step(self, image: torch.Tensor, mask: Optional[torch.Tensor], objects: Optional[List[int]], *, idx_mask: bool,
              end: bool, delete_buffer: bool, force_permanent: bool, next_image: Optional[torch.Tensor]) -> torch.Tensor:
        src_id = image               # the caller's tensor itself: a look-ahead hit is decided on its memory + version
        if objects is None and mask is not None:
            assert not idx_mask
            objects = list(range(1, mask.shape[0] + 1))

        # optional internal down-scaling (the GUI / demo path)
        resize_needed = False
        if self.max_internal_size > 0:
            h, w = image.shape[-2:]
            short = min(h, w)
            if short > self.max_internal_size:
                resize_needed = True
                new_hw = (int(h / short * self.max_internal_size), int(w / short * self.max_internal_size))
                image = F.interpolate(image[None], size=new_hw, mode='bilinear', align_corners=False)[0]
                if mask is not None:
                    if idx_mask:
                        mask = F.interpolate(mask[None, None].float(), size=new_hw,
                                             mode='nearest-exact')[0, 0].round().long()
                    else:
                        mask = F.interpolate(mask[None], size=new_hw, mode='bilinear', align_corners=False)[0]

        self.curr_ti += 1
        image, self.pad = pad_divide_by(image, 16)
        image = image.unsqueeze(0)
        if self.flip_aug:
            image = torch.cat([image, torch.flip(image, dims=[-1])], dim=0)

        since_mem = self.curr_ti - self.last_mem_ti
        is_mem_frame = (since_mem >= self.mem_every or mask is not None) and not end
        need_segment = mask is None or (self.object_manager.num_obj > 0 and not self.object_manager.has_all(objects))
        update_sensory = (since_mem in self.stagger_ti) and not end

        if self.use_cuda_graphs and _graphable(image) and not self.flip_aug:
            if self._graphs is None:
                from cutie_b200.inference.frame_graphs import FrameGraphs
                self._graphs = FrameGraphs(self.network)
            if self._lookahead is None:
                self._lookahead = EncoderLookahead(self._encode_graph)
            (ms_feat, pix_feat, key, shrinkage, selection), _hit = self._lookahead.current(self.curr_ti, image, src_id,
                                                                                          mode=self._amp)
            if next_image is not None and _graphable(next_image) and not resize_needed:
                self._encode_ahead(next_image)
        else:
            ms_feat, pix_feat = self.image_feature_store.get_features(self.curr_ti, image)
            key, shrinkage, selection = self.image_feature_store.get_key(self.curr_ti, image)
        if self.object_shards is not None:
            # every rank's top-k, usage and memory keys follow rank 0's keys: the replicated state stays identical even
            # where a library call (e.g. an autotuned cuDNN convolution of the encoder) rounds differently on some rank
            key, shrinkage, selection = self.object_shards.broadcast((key, shrinkage, selection))

        if need_segment:
            prob_with_bg = self._segment(key, selection, pix_feat, ms_feat, update_sensory=update_sensory)

        if mask is not None:
            tmp_ids, _ = self.object_manager.add_new_objects(objects)
            if self.object_shards is not None:
                self.object_shards.add(self.object_manager.all_obj_ids)
            mask, _ = pad_divide_by(mask, 16)
            if need_segment:
                # merge the propagated prediction with the (partial) input mask; input wins where it is set
                prob_no_bg = prob_with_bg[1:]
                if idx_mask:
                    prob_no_bg[:, mask > 0] = 0
                else:
                    prob_no_bg[:, mask.max(0) > 0.5] = 0
                extra = []
                for mask_pos, tmp_id in enumerate(tmp_ids):
                    plane = (mask == objects[mask_pos]).type_as(prob_no_bg) if idx_mask else mask[tmp_id]
                    if tmp_id > prob_no_bg.shape[0]:
                        extra.append(plane.unsqueeze(0))
                    else:
                        prob_no_bg[tmp_id - 1] = plane
                mask = torch.cat([prob_no_bg, *extra], dim=0)
            elif idx_mask:
                if len(objects) == 0:
                    if delete_buffer:
                        self.image_feature_store.delete(self.curr_ti)
                    log.warning('Trying to insert an empty mask as memory!')
                    return torch.zeros((1, key.shape[-2] * 16, key.shape[-1] * 16), device=key.device,
                                       dtype=key.dtype)
                mask = torch.stack([mask == objects[i] for i, _ in enumerate(tmp_ids)], dim=0)
            prob_with_bg = torch.softmax(aggregate(mask, dim=0), dim=0)

        self.last_mask = prob_with_bg[1:].unsqueeze(0)
        if self.flip_aug:
            self.last_mask = torch.cat([self.last_mask, torch.flip(self.last_mask, dims=[-1])], dim=0)

        if is_mem_frame or force_permanent:
            self._add_memory(image, pix_feat, self.last_mask, key, shrinkage, selection,
                             force_permanent=force_permanent)

        if delete_buffer:
            self.image_feature_store.delete(self.curr_ti)

        out = unpad(prob_with_bg, self.pad)
        if resize_needed:
            out = F.interpolate(out[None], size=(h, w), mode='bilinear', align_corners=False)[0]
        return out

    def _encode_graph(self, image: torch.Tensor, slot: int):
        with K_._call('region:encode_graph', 0):
            return self._graphs.encode(image, slot, amp=self._amp)

    def _encode_ahead(self, next_image: torch.Tensor) -> None:
        """Enqueue G1 (image encoder + key projection) of the next frame on the side stream (EncoderLookahead.ahead);
        this frame's own work is enqueued on the current stream after this call and runs concurrently with it."""
        if self.max_internal_size > 0 and min(next_image.shape[-2:]) > self.max_internal_size:
            return                                    # the internal down-scaling path recomputes on the main stream
        self._lookahead.ahead(self.curr_ti, next_image, lambda t: pad_divide_by(t, 16)[0].unsqueeze(0), mode=self._amp)

    def delete_objects(self, objects: List[int]) -> None:
        self.object_manager.delete_objects(objects)
        self.memory.purge_except(self.object_manager.all_obj_ids)
        if self.object_shards is not None:
            self.object_shards.retain(self.object_manager.all_obj_ids)

    def output_prob_to_mask(self, output_prob: torch.Tensor) -> torch.Tensor:
        """argmax over channels, then tmp-id -> object-id remap (one fused kernel on the GPU)."""
        prob = output_prob.float()
        if prob.stride(-1) != 1:
            prob = prob.contiguous()
        return K_.prob_to_mask(prob, self.object_manager.tmp_to_obj_lut(prob.device))
