"""Object transformer on fused sm_90a kernels (SURVEY.md section 8 rows a9-a15).

Same parameters / state_dict names / call signature as the reference's QueryTransformer
(cutie/model/transformer/object_transformer.py:76-205, transformer_layers.py:12-136), different
execution plan:

  * all pixel-side tensors stay channel-major [B*K, E, HW] for the whole stack -- no NCHW<->NLC
    round trips (the reference does two per block, object_transformer.py:50, transformer_layers.py:131);
  * nn.MultiheadAttention is never instantiated.  Both cross attentions are algebraically folded so
    that the per-pixel K/V (read_from_pixel) and Q/out (read_from_query) projections disappear:
        read_from_pixel : scores = (Q_h Wk_h) . (pix+pe)  ;  out_h = (P_h . pix) Wv_h^T + bv_h
        read_from_query : scores = (pix+pe) . (K_h Wq_h)^T + K_h.bq_h ;  out = pix + P . (V_h Wo_h^T) + bo
    (the key-side bias of read_from_pixel is constant over the softmax axis and drops out);
  * the boolean attention mask [(B*K*heads), Q, HW] is never materialised: a 1-byte-per-pixel
    foreground map + per-object foreground count describe it completely (SURVEY.md Appendix A);
  * LayerNorm / positional add / bias / ReLU / residual are fused into the skinny linear kernel.

The 1x1 projections and the 3x3 PixelFFN convolutions remain cuDNN calls (section 8(f).1, "next").
"""
import math
import os
from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from cutie_b200 import kernels as K_
from cutie_b200.model.blocks import ChannelAttnResBlock, ObjConv2d
from cutie_b200.model.positional import SinusoidPE


# The query-side ops between the tensor-core cross attentions can run as one persistent launch per block (cutie_qt_chain,
# csrc/qt.cu: bit-identical to the separate launches).  On the earlier Blackwell build the 4 chain
# launches measured slower than the 44 separate launches they replace (the separate kernels' few microseconds are
# dependent-load latency, not launch overhead), and a persistent grid of one CTA per SM runs the 384- and
# 1152-tile ops (merge, FFN 1, head folds) in several latency-bound rounds where separate launches run them in one wave.
# So the committed plan is the separate launches; the chain stays selectable (environment variable, echoed by bench.py in
# `build.qt_chain`) as the alternative and is kept under test (not re-measured on H100).
QT_CHAIN = os.environ.get('CUTIE_B200_QT_CHAIN', '0') == '1'


class PackedAttentionParams(nn.Module):
    """Parameter holder with nn.MultiheadAttention's state_dict layout (in_proj_weight [3E,E], ...)."""

    def __init__(self, dim: int):
        super().__init__()
        self.in_proj_weight = nn.Parameter(torch.empty(3 * dim, dim))
        self.in_proj_bias = nn.Parameter(torch.zeros(3 * dim))
        self.out_proj = nn.Linear(dim, dim)
        nn.init.xavier_uniform_(self.in_proj_weight)

    def split(self):
        E = self.out_proj.in_features
        w, b = self.in_proj_weight, self.in_proj_bias
        return (w[:E], w[E:2 * E], w[2 * E:]), (b[:E], b[E:2 * E], b[2 * E:])


class _CrossAttnParams(nn.Module):
    def __init__(self, dim: int, norm: bool):
        super().__init__()
        self.cross_attn = PackedAttentionParams(dim)
        self.norm = nn.LayerNorm(dim) if norm else nn.Identity()


class _SelfAttnParams(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.self_attn = PackedAttentionParams(dim)
        self.norm = nn.LayerNorm(dim)


class _FFNParams(nn.Module):
    def __init__(self, dim: int, ff: int):
        super().__init__()
        self.linear1 = nn.Linear(dim, ff)
        self.linear2 = nn.Linear(ff, dim)
        self.norm = nn.LayerNorm(dim)


class _PixelFFN(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.conv = ChannelAttnResBlock(dim, dim)


class QueryTransformerBlock(nn.Module):
    def __init__(self, model_cfg):
        super().__init__()
        c = model_cfg.object_transformer
        for name in ('read_from_pixel', 'query_self_attention', 'read_from_query'):
            if list(c[name].add_pe_to_qkv) != [True, True, False]:
                raise NotImplementedError('fused kernels implement add_pe_to_qkv=[True, True, False] (model/base.yaml)')
        if c.read_from_query.output_norm:
            raise NotImplementedError('read_from_query.output_norm=True is not implemented by the fused kernels')
        E = c.embed_dim
        self.num_heads, self.num_queries = c.num_heads, c.num_queries
        self.read_from_pixel = _CrossAttnParams(E, norm=True)
        self.self_attn = _SelfAttnParams(E)
        self.ffn = _FFNParams(E, c.ff_dim)
        self.read_from_query = _CrossAttnParams(E, norm=False)
        self.pixel_ffn = _PixelFFN(E)

    def forward(self, x, pixel, query_pe, pixel_pe, fg, fg_count, hw):
        """x, query_pe [M, E]; pixel, pixel_pe [BK, E, HW] channel-major; returns (x, pixel)."""
        H, Q = self.num_heads, self.num_queries
        E = x.shape[1]
        scale = 1.0 / math.sqrt(E // H)
        # --- read_from_pixel (transformer_layers.py:66-98): masked cross attention, queries <- pixels
        rp = self.read_from_pixel
        (wq, wk, wv), (bq, bk, bv) = rp.cross_attn.split()
        xhat = torch.empty_like(x)
        qp = K_.qt_linear(x, wq, bq, ln=(rp.norm.weight, rp.norm.bias), pe=query_pe, xhat_out=xhat)
        qfold, _ = K_.qt_head_fold(qp, wk, transpose_w=False, scale=scale, num_heads=H)
        attn = K_.qt_pixel_to_query(qfold, pixel, pixel_pe, fg, fg_count, wv, bv, Q, H)
        x = K_.qt_linear(attn, rp.cross_attn.out_proj.weight, rp.cross_attn.out_proj.bias, residual=xhat)
        # --- query self attention (transformer_layers.py:27-41)
        sa = self.self_attn
        xhat = torch.empty_like(x)
        qk = K_.qt_linear(x, sa.self_attn.in_proj_weight[:2 * E], sa.self_attn.in_proj_bias[:2 * E],
                          ln=(sa.norm.weight, sa.norm.bias), pe=query_pe, xhat_out=xhat)
        v = K_.qt_linear(xhat, sa.self_attn.in_proj_weight[2 * E:], sa.self_attn.in_proj_bias[2 * E:])
        attn = K_.qt_self_attention(qk, v, Q, H)
        x = K_.qt_linear(attn, sa.self_attn.out_proj.weight, sa.self_attn.out_proj.bias, residual=xhat)
        # --- query FFN (transformer_layers.py:113-118)
        f = self.ffn
        hdn = K_.qt_linear(x, f.linear1.weight, f.linear1.bias, ln=(f.norm.weight, f.norm.bias), relu=True)
        x = K_.qt_linear(hdn, f.linear2.weight, f.linear2.bias, residual=x)
        # --- read_from_query (pixels <- queries), fused through the output projection + residual
        rq = self.read_from_query
        (wq, wk, wv), (bq, bk, bv) = rq.cross_attn.split()
        kp = K_.qt_linear(x, wk, bk, pe=query_pe)
        vp = K_.qt_linear(x, wv, bv)
        kfold, kdots = K_.qt_head_fold(kp, wq, transpose_w=False, scale=scale, bias_vec=bq, num_heads=H)
        vfold, _ = K_.qt_head_fold(vp, rq.cross_attn.out_proj.weight, transpose_w=True, scale=1.0, num_heads=H)
        pixel = K_.qt_query_to_pixel(kfold, kdots, vfold, rq.cross_attn.out_proj.bias, pixel, pixel_pe, Q, H)
        # --- PixelFFN (transformer_layers.py:127-136): cuDNN 3x3 convs, already channel-major
        BK = pixel.shape[0]
        pixel = self.pixel_ffn.conv(pixel.view(BK, E, *hw)).reshape(BK, E, -1).contiguous()
        return x, pixel


class QueryTransformer(nn.Module):
    def __init__(self, model_cfg):
        super().__init__()
        c = model_cfg.object_transformer
        E = c.embed_dim
        self.value_dim, self.embed_dim = model_cfg.value_dim, E
        self.num_heads, self.num_queries, self.num_blocks = c.num_heads, c.num_queries, c.num_blocks
        self.query_init = nn.Embedding(self.num_queries, E)
        self.query_emb = nn.Embedding(self.num_queries, E)
        self.summary_to_query_init = nn.Linear(E, E)
        self.summary_to_query_emb = nn.Linear(E, E)
        self.pixel_init_proj = ObjConv2d(E, E, 1)
        self.pixel_emb_proj = ObjConv2d(E, E, 1)
        self.spatial_pe = SinusoidPE(E, model_cfg.pixel_pe_scale, model_cfg.pixel_pe_temperature)
        self.blocks = nn.ModuleList(QueryTransformerBlock(model_cfg) for _ in range(self.num_blocks))
        self.mask_pred = nn.ModuleList(nn.Sequential(nn.ReLU(), ObjConv2d(E, 1, 1))
                                       for _ in range(self.num_blocks + 1))

    def _aux(self, i: int, pixel_cm: torch.Tensor, B: int, K: int, objects=None):
        """mask_pred[i] + the foreground test.  With `objects` (an object_shards.ObjectGroup: `pixel_cm` holds its
        local objects) the test runs against the logits of all the group's objects, all-gathered from their owners.
        forward() calls this once per head of mask_pred, in order: exchange_without_objects relies on it."""
        conv = self.mask_pred[i][1]
        if objects is None:
            return K_.qt_aux_mask(pixel_cm, conv.weight.view(-1), conv.bias, B, K)
        logits = K_.qt_mask_logits(pixel_cm, conv.weight.view(-1), conv.bias, B, K)
        fg, cnt = K_.qt_aux_fg(objects.gather(logits), objects.positions_tensor(logits.device))
        return logits, fg, cnt

    def exchange_without_objects(self, objects, B: int, hw: int, device) -> None:
        """A rank that owns none of `objects` joins the all-gather of every _aux call forward() makes (one per head of
        mask_pred), contributing no rows, so that the ranks' collectives stay in step."""
        for _ in self.mask_pred:
            objects.gather(torch.empty(B, 0, hw, device=device))

    def forward(self, pixel: torch.Tensor, obj_summaries: torch.Tensor, selector: Optional[torch.Tensor] = None,
                need_weights: bool = False, *, objects=None):
        """pixel [B,K,E,h,w]; obj_summaries [B,K,T,Q,E+1] -> (pixel [B,K,E,h,w], aux dict)
        (object_transformer.py:114-177).  `selector` (training-time object padding) and `need_weights`
        (attention-map export) are not part of the inference hot path and are rejected.
        objects (extension; object sharding): the object_shards.ObjectGroup of the objects whose foreground tests
        couple; `pixel` holds this rank's objects of it."""
        if selector is not None or need_weights or self.training:
            raise NotImplementedError('cutie_b200 implements the inference path (selector=None, need_weights=False)')
        B, K, E, h, w = pixel.shape
        T, Q = obj_summaries.shape[2], self.num_queries
        if T != 1:
            obj_summaries = obj_summaries.sum(dim=2, keepdim=True)      # sums and areas both add (:128-131)
        summ = obj_summaries.reshape(B * K * Q, E + 1).contiguous()
        if QT_CHAIN and (h * w + 63) // 64 <= K_.QT_CHAIN_MAX_TILES:
            return self._forward_chained(pixel, summ, objects)
        x = K_.qt_linear(summ, self.summary_to_query_init.weight, self.summary_to_query_init.bias,
                         summary_norm=True, residual=self.query_init.weight, residual_mod=Q)
        query_pe = K_.qt_linear(summ, self.summary_to_query_emb.weight, self.summary_to_query_emb.bias,
                                summary_norm=True, residual=self.query_emb.weight, residual_mod=Q)
        # 1x1 projections (cuDNN) and the positional map; everything stays [BK, E, HW]
        # .contiguous(): upstream convolutions may hand over channels-last strides; the kernels read channel-major
        pix = self.pixel_init_proj(pixel).reshape(B * K, E, h * w).contiguous()
        pe = self.spatial_pe.grid(h, w).reshape(h * w, E).t()                     # [E, HW]
        pixel_pe = (self.pixel_emb_proj(pixel).reshape(B * K, E, h * w) + pe).contiguous()

        # one _aux call per head of mask_pred (exchange_without_objects mirrors these under object sharding)
        logits, fg, cnt = self._aux(0, pix, B, K, objects)
        aux_logits = [logits.view(B, K, h, w)]
        for i, blk in enumerate(self.blocks):
            x, pix = blk(x, pix, query_pe, pixel_pe, fg, cnt, (h, w))
            logits, fg, cnt = self._aux(i + 1, pix, B, K, objects)                 # :164-167 (always taken)
            aux_logits.append(logits.view(B, K, h, w))
        return self._finish(pix, aux_logits, fg, B, K, E, h, w)

    def _finish(self, pix, aux_logits, fg, B, K, E, h, w):
        aux: Dict[str, object] = {'logits': aux_logits, 'q_weights': None, 'p_weights': None,
                                  'fg_map': fg.view(B, K, h, w)}
        return pix.view(B, K, E, h, w), aux

    def _forward_chained(self, pixel: torch.Tensor, summ: torch.Tensor, objects=None):
        """forward() with the query-side ops fused: one cutie_qt_chain launch for the query initialisation and block 0's
        query projection, then per block [read_from_pixel tiles on wgmma] -> ONE chain (merge + value projection,
        out-proj, self attention, FFN, this block's key/value folds and the NEXT block's query fold) -> [read_from_query on
        wgmma] -> PixelFFN.  Same ops, same arguments, same arithmetic as QueryTransformerBlock.forward: 4 launches
        instead of 41 on the query side."""
        B, K, E, h, w = pixel.shape
        Q, H = self.num_queries, self.num_heads
        BK = B * K
        scale = 1.0 / math.sqrt(E // H)

        def q_side(ch, blk, x, query_pe):
            """read_from_pixel's query projection (LayerNorm + pe) in the current phase; returns what the fold needs."""
            (wq, wk, _), (bq, _, _) = blk.read_from_pixel.cross_attn.split()
            rp = blk.read_from_pixel
            qp, xhat = ch.linear(x, wq, bq, ln=(rp.norm.weight, rp.norm.bias), pe=query_pe, want_xhat=True)
            return qp, xhat, wk

        ch = K_.QtChain()
        x = ch.linear(summ, self.summary_to_query_init.weight, self.summary_to_query_init.bias, summary_norm=True,
                      residual=self.query_init.weight, residual_mod=Q)
        query_pe = ch.linear(summ, self.summary_to_query_emb.weight, self.summary_to_query_emb.bias, summary_norm=True,
                             residual=self.query_emb.weight, residual_mod=Q)
        ch.barrier()
        qp, xhat, wk0 = q_side(ch, self.blocks[0], x, query_pe)
        ch.barrier()
        qfold, _ = ch.head_fold(qp, wk0, transpose_w=False, scale=scale, num_heads=H)
        ch.run()

        pix = self.pixel_init_proj(pixel).reshape(BK, E, h * w).contiguous()
        pe = self.spatial_pe.grid(h, w).reshape(h * w, E).t()                     # [E, HW]
        pixel_pe = (self.pixel_emb_proj(pixel).reshape(BK, E, h * w) + pe).contiguous()
        # one _aux call per head of mask_pred (exchange_without_objects mirrors these under object sharding)
        logits, fg, cnt = self._aux(0, pix, B, K, objects)
        aux_logits = [logits.view(B, K, h, w)]
        for i, blk in enumerate(self.blocks):
            rp, sa, f, rq = blk.read_from_pixel, blk.self_attn, blk.ffn, blk.read_from_query
            (_, _, wv), (_, _, bv) = rp.cross_attn.split()
            ws, tiles = K_.qt_pixel_to_query_tiles(qfold, pix, pixel_pe, fg, cnt, Q, H)
            ch = K_.QtChain()
            attn = ch.p2q_combine(ws, tiles, wv, bv, BK, Q, H)
            ch.barrier()
            x = ch.linear(attn, rp.cross_attn.out_proj.weight, rp.cross_attn.out_proj.bias, residual=xhat)
            ch.barrier()
            # self attention (transformer_layers.py:27-41); the value projection re-derives LayerNorm(x) itself (same code,
            # same values) so that it shares the phase of the q/k projection
            ln = (sa.norm.weight, sa.norm.bias)
            qk, xhat2 = ch.linear(x, sa.self_attn.in_proj_weight[:2 * E], sa.self_attn.in_proj_bias[:2 * E], ln=ln,
                                  pe=query_pe, want_xhat=True)
            v = ch.linear(x, sa.self_attn.in_proj_weight[2 * E:], sa.self_attn.in_proj_bias[2 * E:], ln=ln)
            ch.barrier()
            attn = ch.self_attention(qk, v, Q, H)
            ch.barrier()
            x = ch.linear(attn, sa.self_attn.out_proj.weight, sa.self_attn.out_proj.bias, residual=xhat2)
            ch.barrier()
            hdn = ch.linear(x, f.linear1.weight, f.linear1.bias, ln=(f.norm.weight, f.norm.bias), relu=True)
            ch.barrier()
            x = ch.linear(hdn, f.linear2.weight, f.linear2.bias, residual=x)
            ch.barrier()
            (wq, wk, wv2), (bq, bk, bv2) = rq.cross_attn.split()
            kp = ch.linear(x, wk, bk, pe=query_pe)
            vp = ch.linear(x, wv2, bv2)
            nxt = self.blocks[i + 1] if i + 1 < len(self.blocks) else None
            if nxt is not None:
                qp, xhat, wk_next = q_side(ch, nxt, x, query_pe)
            ch.barrier()
            kfold, kdots = ch.head_fold(kp, wq, transpose_w=False, scale=scale, bias_vec=bq, num_heads=H)
            vfold, _ = ch.head_fold(vp, rq.cross_attn.out_proj.weight, transpose_w=True, scale=1.0, num_heads=H)
            if nxt is not None:
                qfold, _ = ch.head_fold(qp, wk_next, transpose_w=False, scale=scale, num_heads=H)
            ch.run()
            pix = K_.qt_query_to_pixel(kfold, kdots, vfold, rq.cross_attn.out_proj.bias, pix, pixel_pe, Q, H)
            pix = blk.pixel_ffn.conv(pix.view(BK, E, h, w)).reshape(BK, E, -1).contiguous()
            logits, fg, cnt = self._aux(i + 1, pix, B, K, objects)                 # :164-167 (always taken)
            aux_logits.append(logits.view(B, K, h, w))
        return self._finish(pix, aux_logits, fg, B, K, E, h, w)

    def attn_mask_from_fg(self, fg: torch.Tensor) -> torch.Tensor:
        """Expand the 1-byte foreground map to the reference's boolean mask layout
        [(B*K*heads), Q, HW] (object_transformer.py:193-205) -- for save_aux / debugging only."""
        B, K, h, w = fg.shape
        f = fg.reshape(B * K, 1, h * w).bool()
        half = self.num_queries // 2
        blocked = torch.cat([(~f).expand(-1, half, -1), f.expand(-1, half, -1)], 1).clone()
        blocked[blocked.all(-1)] = False
        return blocked.repeat_interleave(self.num_heads, dim=0)
