"""CUTIE network root: same constructor, method names, return conventions and state_dict keys as the
reference (cutie/model/cutie.py:18-260) so checkpoints and InferenceCore callers carry over.

Hot-path entry points on the model side are pixel_fusion (a8, cuDNN) and readout_query (a9, fused
kernels).  encode_image / transform_key / encode_mask / segment are the PyTorch/cuDNN stages either
side of the path.
"""
import logging
from typing import Dict, Iterable, List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from cutie_b200 import kernels as K_
from cutie_b200.model.blocks import ObjConv2d, area_resize
from cutie_b200.model.encoders import KeyProjection, MaskDecoder, MaskEncoder, PixelEncoder, PixelFeatureFuser
from cutie_b200.model.object_summarizer import ObjectSummarizer
from cutie_b200.model.object_transformer import QueryTransformer
from cutie_b200.utils.tensor_utils import aggregate

log = logging.getLogger()


def _local(x: Optional[torch.Tensor], objects) -> Optional[torch.Tensor]:
    """The rows of this rank's objects of `objects` (object_shards.ObjectGroup) along the object axis (dim 1)."""
    return None if x is None else x[:, objects.positions]


class _SensoryAuxHead(nn.Module):
    """Training-time auxiliary head (cutie/model/aux_modules.py:14-27); kept so checkpoints load 1:1."""

    def __init__(self, x_dim: int, pix_dim: int):
        super().__init__()
        self.projection = ObjConv2d(x_dim, pix_dim + 1, 1)

    def forward(self, pix_feat, x):
        x = self.projection(x)
        return (pix_feat.unsqueeze(1) * x[:, :, :-1]).sum(2) + x[:, :, -1]


class AuxComputer(nn.Module):
    def __init__(self, cfg):
        super().__init__()
        m = cfg.model
        self.use_query_aux = m.aux_loss.query.enabled
        self.sensory_aux = _SensoryAuxHead(m.sensory_dim, m.embed_dim) if m.aux_loss.sensory.enabled else None

    def forward(self, pix_feat, aux_input, selector):
        def agg(lg, sel):
            p = torch.sigmoid(lg)
            return aggregate(p if sel is None else p * sel, dim=1)
        out = {'attn_mask': aux_input['attn_mask']}
        if self.sensory_aux is not None:
            out['sensory_logits'] = agg(self.sensory_aux(pix_feat, aux_input['sensory']), selector)
        if self.use_query_aux and aux_input['q_logits'] is not None:
            out['q_logits'] = agg(torch.stack(aux_input['q_logits'], 2),
                                  selector.unsqueeze(2) if selector is not None else None)
        return out


class CUTIE(nn.Module):
    def __init__(self, cfg, *, single_object: bool = False):
        super().__init__()
        self.cfg = cfg
        m = cfg.model
        self.ms_dims = m.pixel_encoder.ms_dims
        self.key_dim, self.value_dim = m.key_dim, m.value_dim
        self.sensory_dim, self.pixel_dim, self.embed_dim = m.sensory_dim, m.pixel_dim, m.embed_dim
        self.single_object = single_object
        self.object_transformer_enabled = m.object_transformer.num_blocks > 0

        self.pixel_encoder = PixelEncoder(m)
        self.pix_feat_proj = nn.Conv2d(self.ms_dims[0], self.pixel_dim, 1)
        self.key_proj = KeyProjection(m)
        self.mask_encoder = MaskEncoder(m, single_object=single_object)
        self.mask_decoder = MaskDecoder(m)
        self.pixel_fuser = PixelFeatureFuser(m, single_object=single_object)
        if self.object_transformer_enabled:
            self.object_transformer = QueryTransformer(m)
            self.object_summarizer = ObjectSummarizer(m)
        self.aux_computer = AuxComputer(cfg)
        self.register_buffer('pixel_mean', torch.tensor(list(m.pixel_mean), dtype=torch.float32).view(-1, 1, 1), False)
        self.register_buffer('pixel_std', torch.tensor(list(m.pixel_std), dtype=torch.float32).view(-1, 1, 1), False)

    # -- helpers ---------------------------------------------------------------------------
    def _others(self, masks: torch.Tensor) -> Optional[torch.Tensor]:
        """cutie.py:49-59: for each object the clamped sum of all the other objects' masks."""
        if self.single_object:
            return None
        if masks.shape[1] == 0:
            return torch.zeros_like(masks)
        return (masks.sum(1, keepdim=True) - masks).clamp(0, 1)

    def _normalise(self, image):
        return (image - self.pixel_mean) / self.pixel_std

    # -- stages before the hot path --------------------------------------------------------
    def encode_image(self, image: torch.Tensor) -> (Iterable[torch.Tensor], torch.Tensor):
        ms = self.pixel_encoder(self._normalise(image))
        return ms, self.pix_feat_proj(ms[0])

    def transform_key(self, final_pix_feat, *, need_sk: bool = True, need_ek: bool = True):
        return self.key_proj(final_pix_feat, need_s=need_sk, need_e=need_ek)

    def encode_mask(self, image, ms_features, sensory, masks, *, deep_update: bool = True,
                    chunk_size: int = -1, need_weights: bool = False, objects=None):
        """objects (extension; object sharding): an object_shards.ObjectGroup over the objects of `masks`; `sensory`
        and the results are this rank's objects of it, the others-mask is formed from all of `masks`."""
        others = self._others(masks)
        if objects is not None:
            masks, others = _local(masks, objects), _local(others, objects)
        value, new_sensory = self.mask_encoder(self._normalise(image), ms_features, sensory, masks,
                                               others, deep_update=deep_update,
                                               chunk_size=chunk_size)
        if self.object_transformer_enabled:
            summaries, logits = self.object_summarizer(masks, value, need_weights)
        else:
            summaries, logits = None, None
        return value, new_sensory, summaries, logits

    # -- hot path, model side --------------------------------------------------------------
    def pixel_fusion(self, pix_feat, pixel, sensory, last_mask, *, chunk_size: int = -1, objects=None):
        """cutie.py:142-157 (a8).  objects (extension; object sharding): an object_shards.ObjectGroup over the objects
        of `last_mask`; `pixel`, `sensory` and the result are this rank's objects of it."""
        last_mask = area_resize(self, last_mask, sensory.shape[-2:])
        others = self._others(last_mask)
        if objects is not None:
            last_mask, others = _local(last_mask, objects), _local(others, objects)
        return self.pixel_fuser(pix_feat, pixel, sensory, last_mask, others, chunk_size=chunk_size)

    def readout_query(self, pixel_readout, obj_memory, *, selector=None, need_weights: bool = False, objects=None):
        """cutie.py:159-170 (a9).  objects (extension; object sharding): see QueryTransformer.forward."""
        if not self.object_transformer_enabled:
            return pixel_readout, None
        return self.object_transformer(pixel_readout, obj_memory, selector=selector, need_weights=need_weights,
                                       objects=objects)

    def read_memory(self, *args, **kwargs):
        """Training-time dense read (cutie.py:102-140): outside the inference hot path."""
        raise NotImplementedError('read_memory is the training path; inference reads through MemoryManager.read')

    # -- stage after the hot path ----------------------------------------------------------
    def segment(self, ms_image_feat: List[torch.Tensor], memory_readout, sensory, *, selector=None,
                chunk_size: int = -1, update_sensory: bool = True, objects=None):
        """cutie.py:172-203 -> (sensory, logits [B,1+K,16h,16w], prob).
        objects (extension; object sharding): an object_shards.ObjectGroup over all objects.  `memory_readout` and
        `sensory` hold this rank's objects of it (None if it owns none) and so does the returned sensory; the decoder
        logits are all-gathered before the aggregation, so `logits` and `prob` cover every object."""
        if objects is not None and not objects.local_ids:
            f16 = ms_image_feat[0]
            sensory, logits = None, f16.new_empty(f16.shape[0], 0, 4 * f16.shape[-2], 4 * f16.shape[-1])
        else:
            sensory, logits = self.mask_decoder(ms_image_feat, memory_readout, sensory, chunk_size=chunk_size,
                                                update_sensory=update_sensory)
        raw = logits if objects is None else objects.gather(logits)

        def aten():
            prob = torch.sigmoid(raw)
            if selector is not None:
                prob = prob * selector
            lg = F.interpolate(aggregate(prob, dim=1), scale_factor=4, mode='bilinear', align_corners=False)
            return lg, F.softmax(lg, dim=1)
        t = getattr(self, 'glue_dispatch', None)
        if t is None or selector is not None or raw.dim() != 4 or raw.shape[1] + 1 > K_.SEGMENT_TAIL_MAX_CHANNELS:
            lg, prob = aten()
        else:           # sigmoid + aggregate + bilinear x4 + softmax (11 launches) as cutie_segment_tail (2)
            lg, prob = t('segment_tail', (tuple(raw.shape),), aten, lambda trial: K_.segment_tail(raw), raw, rtol=1e-4)
        return sensory, lg, prob

    def compute_aux(self, pix_feat, aux_inputs, selector):
        return self.aux_computer(pix_feat, aux_inputs, selector)

    def forward(self, *args, **kwargs):
        raise NotImplementedError

    def load_weights(self, src_dict: Dict[str, torch.Tensor], init_as_zero_if_needed: bool = False) -> None:
        """cutie.py:212-256: single<->multi object channel surgery, then a non-strict load."""
        src_dict = dict(src_dict)

        def widen(key: str, target_in: int, pad_shape):
            t = src_dict.get(key)
            if t is not None and t.shape[1] == target_in - 1:
                pad = torch.zeros(pad_shape, device=t.device, dtype=t.dtype)
                if not init_as_zero_if_needed:
                    nn.init.orthogonal_(pad)
                log.info(f'Converting {key} from single object to multiple objects.')
                src_dict[key] = torch.cat([t, pad], 1)

        if not self.single_object:
            widen('mask_encoder.conv1.weight', 5, (64, 1, 7, 7))
            widen('pixel_fuser.sensory_compress.weight', self.sensory_dim + 2, (self.value_dim, 1, 1, 1))
        else:
            t = src_dict.get('mask_encoder.conv1.weight')
            if t is not None and t.shape[1] == 5:
                log.warning('Converting mask_encoder.conv1.weight from multiple objects to single object.')
                src_dict['mask_encoder.conv1.weight'] = t[:, :-1]
        own = self.state_dict()
        for k in src_dict:
            if k not in own:
                log.info(f'Key {k} found in src_dict but not in self.state_dict()!!!')
        for k in own:
            if k not in src_dict:
                log.info(f'Key {k} found in self.state_dict() but not in src_dict!!!')
        self.load_state_dict(src_dict, strict=False)

    def optimize_for_inference(self, channels_last: bool = True, fuse_epilogues: bool = True,
                               fuse_glue: bool = True) -> 'CUTIE':
        """Post-load surgery on the PyTorch/cuDNN stages (cutie_b200/model/fuse.py): fold the frozen BatchNorms of
        both ResNet trunks into their convolutions, run the trunks channels-last, and run conv+bias(+residual)(+ReLU)
        epilogues in the form a committed rule names (`fuse.ConvEpilogueFuser`, kept as `self.conv_epilogues`);
        `fuse_glue` lets short ATen chains around the convolutions (area down-sampling, CAResBlock tail, sensory GRU
        gates, ...) run as single cutie_b200 kernels per the committed table of `utils.dispatch` (kept as
        `self.glue_dispatch`).  Deterministic: no run-time timing decides anything.  Numerically equivalent up to fp32
        rounding; the module tree (hence state_dict) of the trunks changes, so call it after load_weights."""
        from cutie_b200.model.fuse import ConvEpilogueFuser, attach_epilogue_fuser, fold_trunk_
        for enc in (self.pixel_encoder, self.mask_encoder):
            fold_trunk_(enc)
            if channels_last:
                for name in ('conv1', 'res2', 'layer1', 'layer2', 'layer3'):
                    m = getattr(enc, name, None)
                    if m is not None:
                        m.to(memory_format=torch.channels_last)
                enc.channels_last = True
        # after the folding: fold_trunk_ replaces the trunk convolutions by new modules
        object.__setattr__(self, 'conv_epilogues', ConvEpilogueFuser(enabled=bool(fuse_epilogues)))
        attach_epilogue_fuser(self, self.conv_epilogues)
        if channels_last and fuse_glue and self.object_transformer_enabled:   # (transformer-less variants: no twins)
            # PixelFFN blocks sit between two of our channel-major kernels: offer a channels-last variant to the trial
            for blk in self.object_transformer.blocks:
                for tw in blk.pixel_ffn.conv.make_channels_last_twins() or ():
                    attach_epilogue_fuser(tw, self.conv_epilogues)
            # so do the decoder's two residual blocks (between cutie_upsample2x_add calls)
            for up in (self.mask_decoder.up_16_8, self.mask_decoder.up_8_4):
                for tw in up.out_conv.make_channels_last_twins():
                    attach_epilogue_fuser(tw, self.conv_epilogues)
        # pixel-side glue (area down-sampling, channel-attention tail, sensory GRU gates): ATen chains vs our kernels
        from cutie_b200.utils.dispatch import GlueDispatch, attach_glue_dispatch
        attach_glue_dispatch(self, GlueDispatch(enabled=bool(fuse_glue)))
        return self

    @property
    def device(self) -> torch.device:
        return self.pixel_mean.device
