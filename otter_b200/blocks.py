"""Block-level forward / backward of the hot path, written explicitly over the C-ABI kernels.

Each block is one torch.autograd.Function whose forward and backward are sequences of
otb_* kernel launches (GEMM with fused epilogues, fused attention, LayerNorm, small passes);
torch autograd only stitches blocks together.  Reference line numbers are for
/root/reference/src/otter_ai/models/otter/modeling_otter.py.
"""
import torch

from . import functional as F
from .params import GradSink, bf16_of, f32_of

BF16 = torch.bfloat16


# Weight-gradient GEMMs only feed the gradient buffers, never the dgrad chain: they are issued on a side stream so
# the small ones (projections, perceiver) overlap the latency-bound kernels of the chain instead of serialising with
# them.  Under CUDA-graph capture the side stream becomes a parallel branch of the graph.  Outputs are allocated on
# the main stream before the fork and the streams re-join before backward returns.
import os as _os

# OTB_XATTN_FUSED=1: the gated block's attention + to_out + gate + residual run as ONE kernel (awaiting its GPU validation)
XATTN_OUT_FUSED = _os.environ.get("OTB_XATTN_FUSED") == "1"
WGRAD_SIDE_STREAM = False   # off: the large wgrads dominate the step, overlap has little to hide
_side = {}


class _WgradStream:
    def __init__(self, device):
        self.on = WGRAD_SIDE_STREAM
        if self.on:
            key = (device.index, torch.cuda.current_stream(device).cuda_stream)
            st = _side.get(key)
            if st is None:
                st = _side[key] = torch.cuda.Stream(device=device)
            self.side, self.main = st, torch.cuda.current_stream(device)

    def run(self, fn):
        """fn() launches wgrad kernels whose inputs are already produced on the main stream."""
        if not self.on:
            return fn()
        self.side.wait_stream(self.main)
        with torch.cuda.stream(self.side):
            fn()

    def join(self):
        if self.on:
            self.main.wait_stream(self.side)


def _as_bf16_2d(t, cols):
    t = t.reshape(-1, cols)
    if t.dtype != BF16:
        t = t.to(BF16)
    return t if t.is_contiguous() else t.contiguous()


# =================================================================================================
# OtterPerceiverBlock  (:129-184)
# =================================================================================================
class PerceiverBlockFn(torch.autograd.Function):
    """(x_media [BT*n1, D], latents [BT*n2, D]) -> latents' [BT*n2, D]"""

    @staticmethod
    def forward(ctx, x, lat, BT, need_dx, heads, nm_w, nm_b, nl_w, nl_b, wq, wkv, wo, ff_w, ff_b, w1, w2):
        D = x.shape[1]
        n1, n2 = x.shape[0] // BT, lat.shape[0] // BT
        inner = heads * 64
        # cat(x, latents) (:166) without a copy: both LayerNorms write into one [media rows | latent rows] buffer,
        # so to_kv is ONE GEMM and the attention kernel reads the two row blocks as its two key sources
        R1, R2 = x.shape[0], lat.shape[0]
        kv_in = torch.empty((R1 + R2, D), device=x.device, dtype=BF16)
        xn, mx, rx = F.layernorm_fwd(x, f32_of(nm_w), f32_of(nm_b), out=kv_in[:R1])        # :159
        ln, ml, rl = F.layernorm_fwd(lat, f32_of(nl_w), f32_of(nl_b), out=kv_in[R1:])      # :161
        q = F.linear_fwd(ln, bf16_of(wq))                                                   # :165
        kv = F.linear_fwd(kv_in, bf16_of(wkv))                                              # :166-167
        kv_x, kv_l = kv[:R1], kv[R1:]
        spec = F.AttnSpec(q, 0, kv_x, 0, inner, BT, heads, n2, n1, 0.125, kv2=kv_l, k2_col0=0, v2_col0=inner, Sk2=n2)
        o, lse = F.attn_fwd(spec)                                                           # :168-179 fused
        lat1 = F.linear_fwd(o, bf16_of(wo), residual=lat)                                   # :180
        h0, mf, rf = F.layernorm_fwd(lat1, f32_of(ff_w), f32_of(ff_b))                      # :182-183
        z = torch.empty((lat.shape[0], w1.shape[0]), device=x.device, dtype=BF16)
        hh = F.linear_fwd(h0, bf16_of(w1), act=1, aux_out=z)
        lat2 = F.linear_fwd(hh, bf16_of(w2), residual=lat1)                                 # :184
        ctx.save_for_backward(x, lat, kv_in, q, kv, o, lse, lat1, h0, z, hh, mx, rx, ml, rl, mf, rf)
        ctx.params = (nm_w, nm_b, nl_w, nl_b, wq, wkv, wo, ff_w, ff_b, w1, w2)
        ctx.cfg = (BT, need_dx, heads, n1, n2, D, inner)
        return lat2

    @staticmethod
    def backward(ctx, dlat2):
        x, lat, kv_in, q, kv, o, lse, lat1, h0, z, hh, mx, rx, ml, rl, mf, rf = ctx.saved_tensors
        nm_w, nm_b, nl_w, nl_b, wq, wkv, wo, ff_w, ff_b, w1, w2 = ctx.params
        BT, need_dx, heads, n1, n2, D, inner = ctx.cfg
        R1 = x.shape[0]
        xn, ln, kv_x, kv_l = kv_in[:R1], kv_in[R1:], kv[:R1], kv[R1:]
        sink = GradSink()
        ws = _WgradStream(x.device)
        dlat2 = _as_bf16_2d(dlat2, D)
        # feed-forward
        g2, acc2 = sink.target(w2)
        ws.run(lambda: F.linear_wgrad(dlat2, hh, out=g2, accumulate=acc2))
        dz = F.linear_dgrad(dlat2, bf16_of(w2), aux_in=z)                       # (dlat2 W2) * gelu'(z)
        g1, acc1 = sink.target(w1)
        ws.run(lambda: F.linear_wgrad(dz, h0, out=g1, accumulate=acc1))
        dh0 = F.linear_dgrad(dz, bf16_of(w1))
        gw, acc = sink.target(ff_w)
        gb, _ = sink.target(ff_b)
        dlat1, _, _ = F.layernorm_bwd(dh0, lat1, mf, rf, f32_of(ff_w), add=dlat2, dgamma=gw, dbeta=gb, accumulate=acc)
        # attention output projection
        go, acco = sink.target(wo)
        ws.run(lambda: F.linear_wgrad(dlat1, o, out=go, accumulate=acco))
        do = F.linear_dgrad(dlat1, bf16_of(wo))
        # fused attention backward
        spec = F.AttnSpec(q, 0, kv_x, 0, inner, BT, heads, n2, n1, 0.125, kv2=kv_l, k2_col0=0, v2_col0=inner, Sk2=n2)
        dq = torch.empty_like(q)
        dkv = torch.empty_like(kv)
        dkv_x, dkv_l = dkv[:R1], dkv[R1:]
        F.attn_bwd(spec, o, 0, lse, do, 0, dq, 0, dkv_x, 0, inner, dkv_l, 0, inner)
        # projections: to_kv's wgrad and dgrad are single GEMMs over the [media | latent] rows
        gq, accq = sink.target(wq)
        gkv, acckv = sink.target(wkv)

        def _proj_wgrads():
            F.linear_wgrad(dq, ln, out=gq, accumulate=accq)
            F.linear_wgrad(dkv, kv_in, out=gkv, accumulate=acckv)

        ws.run(_proj_wgrads)
        dkv_in = F.linear_dgrad(dkv, bf16_of(wkv))                              # [d xn | d ln (kv part)]
        dxn = dkv_in[:R1]
        dln = F.linear_dgrad(dq, bf16_of(wq), residual=dkv_in[R1:])
        # norms
        gw, acc = sink.target(nl_w)
        gb, _ = sink.target(nl_b)
        dlat, _, _ = F.layernorm_bwd(dln, lat, ml, rl, f32_of(nl_w), add=dlat1, dgamma=gw, dbeta=gb, accumulate=acc)
        gw, acc = sink.target(nm_w)
        gb, _ = sink.target(nm_b)
        dx, _, _ = F.layernorm_bwd(dxn, x, mx, rx, f32_of(nm_w), want_dx=need_dx, dgamma=gw, dbeta=gb, accumulate=acc)
        ws.join()
        r = sink.result
        return (dx, dlat, None, None, None, r(nm_w), r(nm_b), r(nl_w), r(nl_b), r(wq), r(wkv), r(wo), r(ff_w),
                r(ff_b), r(w1), r(w2))


# =================================================================================================
# final LayerNorm of the resampler (:235) and latents / frame-emb plumbing (:224-232)
# =================================================================================================
class LayerNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, eps):
        y, m, r = F.layernorm_fwd(x, f32_of(w), f32_of(b), eps)
        ctx.save_for_backward(x, m, r)
        ctx.params = (w, b)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, m, r = ctx.saved_tensors
        w, b = ctx.params
        sink = GradSink()
        gw, acc = sink.target(w)
        gb, _ = sink.target(b)
        dx, _, _ = F.layernorm_bwd(_as_bf16_2d(dy, x.shape[-1]), x, m, r, f32_of(w), dgamma=gw, dbeta=gb,
                                   accumulate=acc)
        return dx.view(x.shape), sink.result(w), sink.result(b), None


class BroadcastRowsFn(torch.autograd.Function):
    """param fp32 [mod, D] -> bf16 [rows, D] with out[r] = param[(r // div) % mod]; grad = grouped column sum."""

    @staticmethod
    def forward(ctx, param, rows, div, mod):
        ctx.param, ctx.cfg = param, (div, mod)
        return F.bcast_rows(f32_of(param).reshape(-1, param.shape[-1]), rows, div, mod)

    @staticmethod
    def backward(ctx, dy):
        p = ctx.param
        div, mod = ctx.cfg
        sink = GradSink()
        g, acc = sink.target(p)
        F.grouped_colsum(_as_bf16_2d(dy, p.shape[-1]), div, mod, out=g.view(-1, p.shape[-1])[:mod], accumulate=acc)
        return sink.result(p), None, None, None


class MediaFromClipFn(torch.autograd.Function):
    """CLIP hidden [n_img, 1+v, D] -> media rows [n_img*v, D] (+ frame_embs[img % F]); grad only to frame_embs."""

    @staticmethod
    def forward(ctx, hidden, frame_embs, F_frames):
        if frame_embs is not None and F_frames > frame_embs.shape[0]:
            raise ValueError(f"{F_frames} frames per media but frame_embs holds max_num_frames={frame_embs.shape[0]} "
                             "(modeling_otter.py:224-226)")
        ctx.fe, ctx.cfg = frame_embs, (F_frames, hidden.shape[1] - 1, hidden.shape[2])
        fe = f32_of(frame_embs) if frame_embs is not None else None
        return F.media_from_clip(hidden, fe, F_frames)

    @staticmethod
    def backward(ctx, dmedia):
        fe = ctx.fe
        Fr, v, D = ctx.cfg
        if fe is None:
            return None, None, None
        sink = GradSink()
        g, acc = sink.target(fe)
        if not acc:
            g.zero_()   # rows >= F of frame_embs receive no gradient
        F.grouped_colsum(_as_bf16_2d(dmedia, D), v, Fr, out=g[:Fr], accumulate=acc)
        return None, sink.result(fe), None


# =================================================================================================
# OtterGatedCrossAttentionBlock (:343-395) incl. OtterMaskedCrossAttention (:238-340)
# =================================================================================================
def masked_cross_attention_fwd(x, media, tt, B, L, Tn, n, T_img, heads, norm_w, norm_b, wq, wkv, wo, *, gate=None,
                               residual=None, want_lse=True, mask_ge=False):
    """Shared by the standalone OtterMaskedCrossAttention module and the gated block.
    Returns (out, saved) where out = (o Wo^T) [* tanh(gate) + residual]."""
    inner = heads * 64
    xn, mx, rx = F.layernorm_fwd(x, f32_of(norm_w), f32_of(norm_b))                           # :283
    q = F.linear_fwd(xn, bf16_of(wq))                                                         # :285
    kv = F.linear_fwd(media, bf16_of(wkv))                                                    # :286-288
    spec = F.AttnSpec(q, 0, kv, 0, inner, B, heads, L, Tn, 0.125, text_time=tt, n_per_media=n, T_img=T_img,
                      mask_ge=mask_ge)
    if gate is not None and residual is not None and XATTN_OUT_FUSED and F.xattn_out_fusable(spec, wo.shape[0]):
        # the north star's single kernel: attention + to_out + tanh gate + residual (csrc/otb_xattn_fused.cu)
        out, a, o, lse = F.xattn_out_fused(spec, bf16_of(wo), f32_of(gate), residual, want_lse=want_lse)
        return out, (xn, mx, rx, q, kv, o, lse, a)
    o, lse = F.attn_fwd(spec, want_lse=want_lse)                                              # :290-333 fused
    a = None
    if gate is not None:
        a = torch.empty((x.shape[0], wo.shape[0]), device=x.device, dtype=BF16)
        out = F.linear_fwd(o, bf16_of(wo), aux_out=a, scale_ptr=f32_of(gate), scale_tanh=True, residual=residual)
    else:
        out = F.linear_fwd(o, bf16_of(wo))                                                    # :340
    return out, (xn, mx, rx, q, kv, o, lse, a)


class MaskedCrossAttentionFn(torch.autograd.Function):
    """Standalone OtterMaskedCrossAttention.forward (:262-340): x [B*L,D], media [B*T*n,Dv] -> [B*L,D]."""

    @staticmethod
    def forward(ctx, x, media, tt, B, L, T_img, n, heads, norm_w, norm_b, wq, wkv, wo, mask_ge=False):
        out, saved = masked_cross_attention_fwd(x, media, tt, B, L, T_img * n, n, T_img, heads, norm_w, norm_b, wq,
                                                wkv, wo, mask_ge=mask_ge)
        xn, mx, rx, q, kv, o, lse, _ = saved
        ctx.save_for_backward(x, media, tt, xn, mx, rx, q, kv, o, lse)
        ctx.params = (norm_w, norm_b, wq, wkv, wo)
        ctx.cfg = (B, L, T_img, n, heads, mask_ge)
        return out

    @staticmethod
    def backward(ctx, dout):
        x, media, tt, xn, mx, rx, q, kv, o, lse = ctx.saved_tensors
        norm_w, norm_b, wq, wkv, wo = ctx.params
        B, L, T_img, n, heads, mask_ge = ctx.cfg
        inner = heads * 64
        sink = GradSink()
        dout = _as_bf16_2d(dout, wo.shape[0])
        g, acc = sink.target(wo)
        F.linear_wgrad(dout, o, out=g, accumulate=acc)
        do = F.linear_dgrad(dout, bf16_of(wo))
        spec = F.AttnSpec(q, 0, kv, 0, inner, B, heads, L, T_img * n, 0.125, text_time=tt, n_per_media=n, T_img=T_img,
                          mask_ge=mask_ge)
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)
        F.attn_bwd(spec, o, 0, lse, do, 0, dq, 0, dkv, 0, inner)
        g, acc = sink.target(wq)
        F.linear_wgrad(dq, xn, out=g, accumulate=acc)
        g, acc = sink.target(wkv)
        F.linear_wgrad(dkv, media, out=g, accumulate=acc)
        dxn = F.linear_dgrad(dq, bf16_of(wq))
        dmedia = F.linear_dgrad(dkv, bf16_of(wkv))
        gw, acc = sink.target(norm_w)
        gb, _ = sink.target(norm_b)
        dx, _, _ = F.layernorm_bwd(dxn, x, mx, rx, f32_of(norm_w), dgamma=gw, dbeta=gb, accumulate=acc)
        r = sink.result
        return dx, dmedia, None, None, None, None, None, None, r(norm_w), r(norm_b), r(wq), r(wkv), r(wo), None


class GatedCrossAttentionBlockFn(torch.autograd.Function):
    """OtterGatedCrossAttentionBlock.forward (:373-395): x [B*L,D], media [B*T*n,Dv] -> [B*L,D]."""

    @staticmethod
    def forward(ctx, x, media, tt, B, L, T_img, n, heads, norm_w, norm_b, wq, wkv, wo, attn_gate, ff_w, ff_b, w1, w2,
                ff_gate, mask_ge=False):
        x1, saved = masked_cross_attention_fwd(x, media, tt, B, L, T_img * n, n, T_img, heads, norm_w, norm_b, wq,
                                               wkv, wo, gate=attn_gate, residual=x, mask_ge=mask_ge)   # :380-389
        xn, mx, rx, q, kv, o, lse, a1 = saved
        h0, mf, rf = F.layernorm_fwd(x1, f32_of(ff_w), f32_of(ff_b))                          # :391-392
        z = torch.empty((x.shape[0], w1.shape[0]), device=x.device, dtype=BF16)
        hh = F.linear_fwd(h0, bf16_of(w1), act=1, aux_out=z)
        a2 = torch.empty_like(x1)
        x2 = F.linear_fwd(hh, bf16_of(w2), aux_out=a2, scale_ptr=f32_of(ff_gate), scale_tanh=True, residual=x1)  # :393
        tt_s = tt if tt is not None else torch.empty(0, device=x.device, dtype=torch.int32)
        ctx.save_for_backward(x, media, tt_s, xn, mx, rx, q, kv, o, lse, a1, x1, h0, mf, rf, z, hh, a2)
        ctx.params = (norm_w, norm_b, wq, wkv, wo, attn_gate, ff_w, ff_b, w1, w2, ff_gate)
        ctx.cfg = (B, L, T_img, n, heads, tt is not None, mask_ge)
        return x2

    @staticmethod
    def backward(ctx, dx2):
        x, media, tt, xn, mx, rx, q, kv, o, lse, a1, x1, h0, mf, rf, z, hh, a2 = ctx.saved_tensors
        norm_w, norm_b, wq, wkv, wo, attn_gate, ff_w, ff_b, w1, w2, ff_gate = ctx.params
        B, L, T_img, n, heads, has_tt, mask_ge = ctx.cfg
        tt = tt if has_tt else None
        D = x.shape[1]
        inner = heads * 64
        sink = GradSink()
        ws = _WgradStream(x.device)
        dx2 = _as_bf16_2d(dx2, D)
        fg, ag = f32_of(ff_gate), f32_of(attn_gate)
        # --- feed-forward branch: y = a2 * tanh(ff_gate) + x1 ---
        g, acc = sink.target(ff_gate)
        F.gate_grad(dx2, a2, fg, dgate=g, accumulate=acc)
        g2, acc2 = sink.target(w2)
        ws.run(lambda: F.linear_wgrad(dx2, hh, out=g2, accumulate=acc2, scale_ptr=fg, scale_tanh=True))
        dz = F.linear_dgrad(dx2, bf16_of(w2), aux_in=z, scale_ptr=fg, scale_tanh=True)
        g1, acc1 = sink.target(w1)
        ws.run(lambda: F.linear_wgrad(dz, h0, out=g1, accumulate=acc1))
        dh0 = F.linear_dgrad(dz, bf16_of(w1))
        gw, acc = sink.target(ff_w)
        gb, _ = sink.target(ff_b)
        dx1, _, _ = F.layernorm_bwd(dh0, x1, mf, rf, f32_of(ff_w), add=dx2, dgamma=gw, dbeta=gb, accumulate=acc)
        # --- attention branch: x1 = a1 * tanh(attn_gate) + x ---
        g, acc = sink.target(attn_gate)
        F.gate_grad(dx1, a1, ag, dgate=g, accumulate=acc)
        go, acco = sink.target(wo)
        ws.run(lambda: F.linear_wgrad(dx1, o, out=go, accumulate=acco, scale_ptr=ag, scale_tanh=True))
        do = F.linear_dgrad(dx1, bf16_of(wo), scale_ptr=ag, scale_tanh=True)
        spec = F.AttnSpec(q, 0, kv, 0, inner, B, heads, L, T_img * n, 0.125, text_time=tt, n_per_media=n, T_img=T_img,
                          mask_ge=mask_ge)
        dq, dkv = torch.empty_like(q), torch.empty_like(kv)
        F.attn_bwd(spec, o, 0, lse, do, 0, dq, 0, dkv, 0, inner)
        gq, accq = sink.target(wq)
        gkv, acckv = sink.target(wkv)

        def _proj_wgrads():
            F.linear_wgrad(dq, xn, out=gq, accumulate=accq)
            F.linear_wgrad(dkv, media, out=gkv, accumulate=acckv)

        ws.run(_proj_wgrads)
        dxn = F.linear_dgrad(dq, bf16_of(wq))
        dmedia = F.linear_dgrad(dkv, bf16_of(wkv)) if ctx.needs_input_grad[1] else None
        gw, acc = sink.target(norm_w)
        gb, _ = sink.target(norm_b)
        dx, _, _ = F.layernorm_bwd(dxn, x, mx, rx, f32_of(norm_w), add=dx1, dgamma=gw, dbeta=gb, accumulate=acc)
        ws.join()
        r = sink.result
        return (dx, dmedia, None, None, None, None, None, None, r(norm_w), r(norm_b), r(wq), r(wkv), r(wo),
                r(attn_gate), r(ff_w), r(ff_b), r(w1), r(w2), r(ff_gate), None)


# =================================================================================================
# CLIP ViT forward (frozen; no backward)   xformers_model/clip.py:50-199,393-446
# =================================================================================================
def clip_vision_forward(pixel_values, W):
    """pixel_values [N,3,H,W]; W: prepared weight dict (see modeling_clip.prepare_clip_weights).
    Returns last_hidden_state bf16 [N, 1+np, D] (no post_layernorm on the hot path, clip.py:430-434)."""
    N = pixel_values.shape[0]
    patch, D, heads = W["patch"], W["D"], W["heads"]
    np_ = (pixel_values.shape[2] // patch) * (pixel_values.shape[3] // patch)
    if np_ + 1 != W["pos"].shape[0]:          # the kernels index the position table unchecked (HF raises the same way)
        raise ValueError(f"Input image size ({pixel_values.shape[2]}*{pixel_values.shape[3]}) doesn't match model "
                         f"({W['pos'].shape[0] - 1} patches of {patch}*{patch}).")
    cols = F.im2col_patches(pixel_values, patch, W["Kpad"])                               # clip.py:74 conv as GEMM
    pe = F.linear_fwd(cols, W["patch_w"])
    h = F.clip_assemble(pe, W["cls"], W["pos"], N, np_)                                   # clip.py:77-80
    S = np_ + 1
    h, _, _ = F.layernorm_fwd(h.view(N * S, D), W["pre_ln_w"], W["pre_ln_b"], W["eps"], want_stats=False)  # :425
    for lw in W["layers"]:                                                                # clip.py:347
        x, _, _ = F.layernorm_fwd(h, lw["ln1_w"], lw["ln1_b"], W["eps"], want_stats=False)    # :178
        qkv = F.linear_fwd(x, lw["qkv_w"], bias=lw["qkv_b"])                              # :106-110 (fused q|k|v)
        spec = F.AttnSpec(qkv, 0, qkv, D, 2 * D, N, heads, S, S, 0.125)
        o, _ = F.attn_fwd(spec, want_lse=False)                                           # :112-128
        h = F.linear_fwd(o, lw["out_w"], bias=lw["out_b"], residual=h)                    # :131,185
        x, _, _ = F.layernorm_fwd(h, lw["ln2_w"], lw["ln2_b"], W["eps"], want_stats=False)    # :188
        x = F.linear_fwd(x, lw["fc1_w"], bias=lw["fc1_b"], act=2)                         # :145-147 quick_gelu
        h = F.linear_fwd(x, lw["fc2_w"], bias=lw["fc2_b"], residual=h)                    # :148,190
    return h.view(N, S, D)
