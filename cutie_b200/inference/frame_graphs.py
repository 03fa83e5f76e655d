"""CUDA graphs for the arena-independent parts of a propagated frame.

A frame through the eager path issues ~550 kernel launches (cuDNN convolutions, ATen elementwise ops and the
object-transformer kernels), which makes `InferenceCore.step` CPU-launch-bound on a fast GPU.  Two regions of the
frame have static shapes and touch no memory-bank pointers, so each is captured once and replayed:

    G1  image -> ResNet-50 pixel encoder -> pix_feat, key / shrinkage / selection      (CUTIE.encode_image, transform_key)
    G2  (visual readout, pix_feat, sensory, last mask, object memory, multi-scale features)
            -> pixel_fusion -> object transformer (fused kernels) -> mask decoder -> probabilities, new sensory

The memory read between them (cutie_affinity_topk + cutie_readout_gather) stays eager: its segment pointers move
whenever the ring advances.  On memory frames the mask encoder + object summarizer (G3) are a third graph; the
append into the arena stays eager.  Graphs are keyed by every
shape/flag they depend on -- including the precision mode (`amp`: the step runs under fp16 autocast, so the model's
tensor-core convolutions take their FP16-operand form; a capture of one mode is never replayed in the other) -- and are
bypassed (eager path) for multi-bucket / chunked / flip-augmented reads.
Enable with `InferenceCore(..., use_cuda_graphs=True)` or `processor.use_cuda_graphs = True`.
"""
import gc
from typing import Dict, Tuple

import torch

from cutie_b200 import kernels as K_


class _Captured:
    def __init__(self, fn, static_inputs):
        self.inputs = static_inputs
        cur = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        side.wait_stream(cur)
        with torch.cuda.stream(side):           # warm-up off the capture stream (cuDNN autotune, lazy inits)
            for _ in range(2):
                fn(*static_inputs)
        cur.wait_stream(side)
        self.graph = torch.cuda.CUDAGraph()
        before = K_.LAUNCH_COUNT
        # Python's cyclic collector is paused while capturing: it may run at any allocation, and a dead reference cycle
        # holding another capture (a discarded InferenceCore: its encoder look-ahead refers back to it) would destroy that
        # CUDA graph and release its memory pool in the middle of this capture, which invalidates it
        # (cudaErrorStreamCaptureInvalidated).  torch.cuda.graph collects only with torch.compiler.config.force_cudagraph_gc.
        gc_on = gc.isenabled()
        gc.disable()
        try:
            with torch.cuda.graph(self.graph):
                self.outputs = fn(*static_inputs)
        finally:
            if gc_on:
                gc.enable()
        self.kernel_launches = K_.LAUNCH_COUNT - before       # cutie_b200 kernels recorded in this graph

    def replay(self):
        self.graph.replay()
        K_.LAUNCH_COUNT += self.kernel_launches
        return self.outputs


class FrameGraphs:
    def __init__(self, network):
        self.net = network
        self._enc: Dict[Tuple, _Captured] = {}
        self._seg: Dict[Tuple, _Captured] = {}
        self._msk: Dict[Tuple, _Captured] = {}

    # ---- G1 ------------------------------------------------------------------------------------
    def encode(self, image: torch.Tensor, slot: int = 0, amp: bool = False):
        """`slot` selects one of several independent captures (own static input and outputs): InferenceCore alternates
        two of them so that the next frame's encoder can run on a side stream while this frame's outputs are in use."""
        key = (tuple(image.shape), image.device, int(slot), bool(amp))
        cap = self._enc.get(key)
        if cap is None:
            static_img = image.clone()

            def fn(img):
                ms, pix = self.net.encode_image(img)
                k, s, e = self.net.transform_key(ms[0])
                return ms, pix, k, s, e
            cap = self._enc[key] = _Captured(fn, (static_img,))
        cap.inputs[0].copy_(image)
        return cap.replay()

    # ---- G2 ------------------------------------------------------------------------------------
    def segment(self, visual, pix_feat, sensory, last_mask, obj_mem, ms_feat, update_sensory: bool, amp: bool = False):
        """All arguments are tensors; visual/pix_feat/ms_feat may already be graph-static (G1 outputs / the gather
        kernel's fixed output buffer).  Returns (new_sensory or None, logits, prob) in static buffers."""
        key = (tuple(visual.shape), tuple(last_mask.shape), bool(update_sensory), visual.device,
               tuple(t.data_ptr() for t in (pix_feat, *ms_feat)), bool(amp))
        cap = self._seg.get(key)
        if cap is None:
            st = (visual.clone(), sensory.clone(), last_mask.clone(), obj_mem.clone())

            def fn(vis, sens, lm, om):
                fused = self.net.pixel_fusion(pix_feat, vis, sens, lm)
                ro, _aux = self.net.readout_query(fused, om)
                new_sens, logits, prob = self.net.segment(ms_feat, ro, sens, update_sensory=update_sensory)
                return new_sens, logits, prob
            cap = self._seg[key] = _Captured(fn, st)
        for dst, src in zip(cap.inputs, (visual, sensory, last_mask, obj_mem)):
            dst.copy_(src)
        return cap.replay()

    # ---- G3 (memory frames) ----------------------------------------------------------------------
    def encode_mask(self, image, pix_feat, sensory, masks, amp: bool = False):
        """CUTIE.encode_mask (mask encoder + deep sensory update + object summarizer) as one replay.
        Returns (value [B,K,CV,h,w], new_sensory, summaries [B,K,Q,E+1]) in static buffers."""
        key = (tuple(image.shape), tuple(masks.shape), image.device, pix_feat.data_ptr(), bool(amp))
        cap = self._msk.get(key)
        if cap is None:
            st = (image.clone(), sensory.clone(), masks.clone())

            def fn(img, sens, msk):
                value, new_sens, summaries, _ = self.net.encode_mask(img, pix_feat, sens, msk)
                return value, new_sens, summaries
            cap = self._msk[key] = _Captured(fn, st)
        for dst, src in zip(cap.inputs, (image, sensory, masks)):
            dst.copy_(src)
        return cap.replay()
