"""Bi-directional image<->text multi-head attention of the VL deep-fusion tower on sm_90a kernels.

Drop-in for maskrcnn_benchmark/utils/fuse_helper.py: ``BiMultiHeadAttention`` (:171-303) and
``BiAttentionBlockForCheckpoint`` (:344-426), same constructor arguments / parameter names / forward signatures,
eval mode (dropout and DropPath are identities).

Layout: the 5 FPN levels are kept concatenated as ONE fp16 tensor v [B, N, 256] (P3->P7, row-major (h, w)) — exactly the
``permute_and_flatten`` + ``cat`` the reference builds at :398-404 — so the tower never converts back to NCHW between
layers (``forward_flat``).  ``forward`` keeps the reference's NCHW-in / NCHW-out signature for drop-in use.

Every product is a K-major x K-major wgmma GEMM; transposed operands are produced by swapping operand roles
(V^T = W . x^T), never by a transpose kernel:
    Q  = (LN(v) Wv^T + b) * d^-1/2      [B,N,E]      K  = LN(l) Wl^T + b          [B,T,E]
    VvT= Wvv LN(v)^T + b (per row)      [B,E,N]      VlT= Wvl LN(l)^T + b         [B,E,T]
    A  = clamp(Q_h K_h^T)  [B,H,N,T] -> softmax_T(A + mask)            -> out_v = P_v VlT_h^T
                                     -> column softmax, transposed    -> out_l = P_l VvT_h^T
    v' = LN(v) + gamma_v * (out_v Wov^T + b)       l' = LN(l) + gamma_l * (out_l Wol^T + b)
"""
import torch
from torch import nn

from .. import ops
from .._lib import VEC_PER_COL, VEC_PER_ROW, MqdetError
from .weights import f32, w16


def _flatten_levels(feats):
    """[B,C,h,w] x L -> [B, sum(hw), C] (permute_and_flatten + cat, fuse_helper.py:398-404). Data movement only."""
    return torch.cat([f.flatten(2).transpose(1, 2) for f in feats], dim=1).contiguous()


def _split_levels(v, sizes):
    """[B,N,C] -> list of [B,C,h,w] (:406-412)."""
    out, start = [], 0
    B, _, C = v.shape
    for (h, w) in sizes:
        out.append(v[:, start:start + h * w].transpose(1, 2).reshape(B, C, h, w).contiguous())
        start += h * w
    return out


class BiMultiHeadAttention(nn.Module):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, dropout=0.1, cfg=None, *, stable_softmax_2d=None,
                 clamp_min_for_underflow=None, clamp_max_for_overflow=None, mask_fill=(-9e15, 1.0)):
        """``cfg`` supplies the three score flags (MODEL.DYHEAD.FUSE_CONFIG) unless they are given explicitly — the
        GroundingDINO variant (modeling/groundingdino/fuse_modules.py) hard-codes them.  ``mask_fill`` = (value added at padded
        text tokens, value added at kept ones): fuse_helper.py:270-283 adds -9e15 / +1, GroundingDINO fills -inf / 0."""
        super().__init__()
        self.embed_dim = embed_dim
        self.num_heads = num_heads
        self.head_dim = embed_dim // num_heads
        self.v_dim, self.l_dim = v_dim, l_dim
        assert self.head_dim * num_heads == embed_dim
        self.scale = self.head_dim ** (-0.5)
        self.dropout = dropout
        self.v_proj = nn.Linear(v_dim, embed_dim)
        self.l_proj = nn.Linear(l_dim, embed_dim)
        self.values_v_proj = nn.Linear(v_dim, embed_dim)
        self.values_l_proj = nn.Linear(l_dim, embed_dim)
        self.out_v_proj = nn.Linear(embed_dim, v_dim)
        self.out_l_proj = nn.Linear(embed_dim, l_dim)
        fc = cfg.MODEL.DYHEAD.FUSE_CONFIG if cfg is not None else None
        # "fused" (default): the product path (_attend_fused); "f32": the score matrices in fp32 in HBM until both softmaxes have
        # been taken, like the reference (fuse_helper.py:240-291) — twice the traffic; the reference the product path is tested
        # against, and the diagnostic mode of tests/test_parity_experiment_gpu.py.  Any other value is an error.
        self.score_precision = "fused"
        self.stable_softmax_2d = bool(fc.STABLE_SOFTMAX_2D if stable_softmax_2d is None else stable_softmax_2d)
        self.clamp_min_for_underflow = bool(fc.CLAMP_MIN_FOR_UNDERFLOW if clamp_min_for_underflow is None else clamp_min_for_underflow)
        self.clamp_max_for_overflow = bool(fc.CLAMP_MAX_FOR_OVERFLOW if clamp_max_for_overflow is None else clamp_max_for_overflow)
        self.mask_fill = (float(mask_fill[0]), float(mask_fill[1]))
        # STABLE_SOFTMAX_2D subtracts the GLOBAL maximum of the score tensor before the clamps (fuse_helper.py:240-242,
        # GroundingDINO fuse_modules.py:177-178): that needs the whole score tensor before either softmax, so it takes the
        # explicit fp32-score path (global_max + shift_clamp kernels) instead of the fused one
        self._reset_parameters()

    def _reset_parameters(self):
        for m in (self.v_proj, self.l_proj, self.values_v_proj, self.values_l_proj, self.out_v_proj, self.out_l_proj):
            nn.init.xavier_uniform_(m.weight)
            m.bias.data.fill_(0)

    SPLIT_K = 8

    def _fused_applies(self, Cv, T):
        """Whether the product path runs: ``score_precision == "fused"``, no STABLE_SOFTMAX_2D (its global maximum needs the
        whole score tensor) and a shape inside the fused kernels' envelope (head dim 256, Cv = 256, T % 8 == 0, T <= 256,
        H <= 8).  Everything else takes the explicit fp32-score path."""
        if self.score_precision not in ("fused", "f32"):
            raise ValueError(f"BiMultiHeadAttention.score_precision must be 'fused' or 'f32', got {self.score_precision!r}")
        return (self.score_precision == "fused" and not self.stable_softmax_2d and self.head_dim == 256 and Cv == 256
                and T % 8 == 0 and T <= 256 and self.num_heads <= 8)

    def _score_clamp(self):
        """The +-5e4 clamp of the scores (fuse_helper.py:245-252) as the kernels take it: 0 = none."""
        return 50000.0 if (self.clamp_min_for_underflow or self.clamp_max_for_overflow) else 0.0

    def _keys(self, ln16):
        """k = LN(l) Wl^T + b  [B,T,H,d] fp16."""
        B, T = ln16.shape[:2]
        return ops.gemm(ln16.view(B * T, -1), w16(self.l_proj.weight), bias=f32(self.l_proj.bias)).view(B, T, self.num_heads,
                                                                                                           self.head_dim)

    @torch.no_grad()
    def _attend(self, vn16, ln16, mask_l, v_epilogue=None, l_epilogue=None, mask_v=None):
        """vn16 [B,N,256] fp16, ln16 [B,T,768] fp16 (already layer-normed), mask_l [B,T] (1 keep / 0 padding) -> (dv, dl).
        ``*_epilogue`` = dict(gate=gamma, residual=normed input) fuses the layer-scale + residual into the out-proj.
        ``mask_v`` [B,N] (1 keep / 0 padding; GroundingDINO's attention_mask_v) only on the explicit fp32-score path."""
        B, N, Cv = vn16.shape
        T = ln16.shape[1]
        if self._fused_applies(Cv, T) and mask_v is None:
            return self._attend_fused(vn16, ln16, mask_l, v_epilogue, l_epilogue)
        H, d, E = self.num_heads, self.head_dim, self.embed_dim
        dev = vn16.device
        k = self._keys(ln16)
        explicit = self.stable_softmax_2d or mask_v is not None
        # explicit path with many image tokens: the text-side P^T.V contracts over N with only B*H*T/128 output tiles, so it runs as
        # SPLIT_K K-slices (an extra GEMM batch dimension) -> N is padded to a multiple of 64 * SPLIT_K instead of 8
        split = self.SPLIT_K if (explicit and N >= 8192) else 1
        Np = (N + 64 * split - 1) // (64 * split) * (64 * split) if split > 1 else (N + 7) // 8 * 8
        q = ops.gemm(vn16.view(B * N, Cv), w16(self.v_proj.weight), bias=f32(self.v_proj.bias), alpha=self.scale,
                     scale_after_bias=True).view(B, N, H, d)
        vvT = torch.empty((B, E, Np), dtype=torch.float16, device=dev)
        if Np != N:
            vvT[:, :, N:].zero_()   # only the K-padding columns (a full memset is 91 MB per layer at N = 22323)
        ops.gemm(w16(self.values_v_proj.weight), vn16, out=vvT[:, :, :N], bias=f32(self.values_v_proj.bias),
                 bias_mode=VEC_PER_ROW)
        vlT = ops.gemm(w16(self.values_l_proj.weight), ln16, bias=f32(self.values_l_proj.bias), bias_mode=VEC_PER_ROW)

        qh, kh = q.permute(0, 2, 1, 3), k.permute(0, 2, 1, 3)
        return self._finish(*self._attend_f32_scores(qh, kh, vvT, vlT, mask_l, self._score_clamp(), B, N, T, Np, mask_v),
                            v_epilogue, l_epilogue, B, N, T, Cv)

    def _query_fold_weights(self):
        """(scale * Wq)^T as fp16 [Cv, E] and scale * bq as fp16 [H, 8, d] (row 0 used), cached per parameter version: the B
        operands that fold the query projection into the keys.  scale = d^-1/2 = 2^-4 for d = 256: exact in fp16."""
        ps = (self.v_proj.weight, self.v_proj.bias)
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if getattr(self, "_qfold", None) is None or self._qfold[0] != key:
            H, d = self.num_heads, self.head_dim
            wt = ops.cast_f16((self.v_proj.weight.detach().float() * self.scale).t().contiguous())        # [Cv, E]
            bq = torch.zeros((H, 8, d), dtype=torch.float32, device=wt.device)
            bq[:, 0] = (self.v_proj.bias.detach().float() * self.scale).view(H, d)
            self._qfold = (key, wt, ops.cast_f16(bq))
        return self._qfold[1], self._qfold[2]

    def _attend_fused(self, vn16, ln16, mask_l, v_epilogue, l_epilogue):
        """Product path: neither the queries q [B,N,E], the score matrix, its transpose, the per-head contexts nor the image-side
        value tensor reach HBM, and the scores stay fp32 until both softmaxes have been taken.  Three per-(image, head)
        operands of [256 x 256] fold the projections into the text side (tiny GEMMs over the T = 256 tokens):
            gT_h = K_h (d^-1/2 Wq_h)            S = (vn Wq_h^T + bq_h) d^-1/2 K_h^T == vn gT_h^T + gbias_h,  gbias_h = d^-1/2 bq_h . K_h
            mT_h = Wout_h Vl_h^T                (P Vl_h) Wout_h^T == P mT_h^T
          image side: ONE kernel = S (registers) -> masked row softmax -> P . mT accumulated over the heads -> layer scale + residual;
                      it also emits the column maxima of the scores;
          text side : ONE kernel = S^T recomputed from gT and the image tokens -> exp(. - column max) -> P^T . vn (the image
                      tokens themselves; the value projection follows as a small per-head GEMM because sum_n p[n] = 1) with
                      in-kernel column sums."""
        dv, ctx = self._fused_image(vn16, ln16, mask_l, v_epilogue)
        return dv, self._fused_text(ctx, l_epilogue)

    def _fused_image(self, vn16, ln16, mask_l, v_epilogue):
        """Image side of the product path (see _attend_fused) -> (dv [B,N,Cv] fp16, context of the text side).  The text side
        only needs that context, so a caller may run it on another stream next to the visual branch (VLDyHead.forward_flat)."""
        B, N, Cv = vn16.shape
        T = ln16.shape[1]
        H, d, E = self.num_heads, self.head_dim, self.embed_dim
        dev = vn16.device
        ve = v_epilogue or {}
        clamp = self._score_clamp()
        kh = self._keys(ln16).permute(0, 2, 1, 3)                                      # [B,H,T,d]
        wqT, bq8 = self._query_fold_weights()
        gT = torch.empty((B, H, T, Cv), dtype=torch.float16, device=dev)
        ops.gemm(kh, wqT.view(1, Cv, H, d).permute(0, 2, 1, 3), out=gT)                # gT[b,h,t,c] = sum_dd K[b,t,h,dd] scale Wq[h*d+dd, c]
        gbias = torch.empty((B, H, T, 8), dtype=torch.float32, device=dev)
        ops.gemm(kh, bq8.view(1, H, 8, d), out=gbias)                                  # column 0 = scale bq_h . K_h[t]
        vl = ops.gemm(ln16.view(B * T, -1), w16(self.values_l_proj.weight), bias=f32(self.values_l_proj.bias)).view(B, T, H, d)
        mT = torch.empty((B, H, Cv, T), dtype=torch.float16, device=dev)
        ops.gemm(w16(self.out_v_proj.weight).view(1, Cv, H, d).permute(0, 2, 1, 3), vl.permute(0, 2, 1, 3), out=mT)
        cm = mask_l.float().contiguous() if mask_l is not None else None
        dv, colmax = ops.biattn_image(vn16, gT, gbias, mT, f32(self.out_v_proj.bias), ve.get("gate"), ve.get("residual"), cm,
                                      clamp, H)
        return dv, dict(gT=gT, gbias=gbias, vn16=vn16, colmax=colmax, clamp=clamp)

    def _fused_text(self, ctx, l_epilogue):
        """Text side of the product path: S^T recomputed from gT and the image tokens, softmax over all image tokens, value
        projection after the token reduction, output projection (+ layer scale + residual) -> dl [B,T,l_dim] fp32."""
        gT, gbias, vn16, colmax, clamp = ctx["gT"], ctx["gbias"], ctx["vn16"], ctx["colmax"], ctx["clamp"]
        B, N, Cv = vn16.shape
        H, d, E = self.num_heads, self.head_dim, self.embed_dim
        T = gT.shape[2]
        dev = vn16.device
        le = l_epilogue or {}
        u = torch.empty((B, H, T, Cv), dtype=torch.float16, device=dev)
        ops.biattn_text_vn(gT, vn16.view(B, 1, N, Cv).expand(B, H, N, Cv), vn16, colmax, clamp, u, rowbias=gbias)
        # out_l[b, t, h, :] = u[b, h, t, :] . Wvv_h^T + b_h   (value projection after the token reduction)
        ol = torch.empty((B, T, H, d), dtype=torch.float16, device=dev)
        ops.gemm(u, w16(self.values_v_proj.weight).view(1, H, d, Cv), out=ol.permute(0, 2, 1, 3),
                 bias=f32(self.values_v_proj.bias).view(H, d))
        dl = ops.gemm(ol.view(B * T, E), w16(self.out_l_proj.weight), bias=f32(self.out_l_proj.bias),
                      out_dtype=torch.float32, gate=le.get("gate"), gate_mode=VEC_PER_COL if le else 0,
                      residual=le["residual"].view(B * T, -1) if le else None)
        return dl.view(B, T, -1)

    def _attend_f32_scores(self, qh, kh, vvT, vlT, mask_l, clamp, B, N, T, Np, mask_v=None):
        """Both score matrices in fp32 (A and its transpose as two products), softmaxes on the fp32 values: the diagnostic
        variant of the GLIP path and THE path of STABLE_SOFTMAX_2D / an image-token mask (GroundingDINO)."""
        H, d = self.num_heads, self.head_dim
        dev = qh.device
        cm = mask_l.float().contiguous() if mask_l is not None else None
        stable = self.stable_softmax_2d
        lim = clamp if clamp > 0 else float("inf")
        A32 = torch.empty((B, H, N, T), dtype=torch.float32, device=dev)
        ops.gemm(qh, kh, out=A32, clamp=0.0 if stable else clamp)
        if stable:  # attn_weights - attn_weights.max(), then the clamps; the maximum stays on the device, the shift + clamps ride in
            gmax = ops.global_max(A32)  # the softmax kernels (no pass of their own over the 183 MB score tensors)
            Pv = ops.softmax_rows_shifted(A32, gmax, -lim, lim, colmask=cm, rows_per_batch=H * N, mask_value=self.mask_fill[0],
                                          keep_add=self.mask_fill[1])
        else:
            Pv = ops.softmax_rows(A32, colmask=cm, rows_per_batch=H * N, mask_value=self.mask_fill[0], keep_add=self.mask_fill[1])
        del A32
        AT32 = torch.empty((B, H, T, Np), dtype=torch.float32, device=dev)
        if Np != N:
            AT32[..., N:].zero_()
        ops.gemm(kh, qh, out=AT32[..., :N], clamp=0.0 if stable else clamp)
        # padded image tokens leave the text side's softmax (fuse_modules.py:201-206); mask rows are indexed with stride n (= N), not
        # with the padded row length (mqdet_softmax_rows)
        mv = mask_v.float().contiguous() if mask_v is not None else None
        mkw = dict(colmask=mv, rows_per_batch=H * T, mask_value=float("-inf"), keep_add=0.0) if mv is not None else {}
        if stable:
            Pl = ops.softmax_rows_shifted(AT32, gmax, -lim, lim, n=N, **mkw)
        else:
            Pl = ops.softmax_rows(AT32, n=N, **mkw)
        del AT32
        ov = torch.empty((B, N, H, d), dtype=torch.float16, device=dev)
        ops.gemm(Pv, vlT.view(B, H, d, T), out=ov.permute(0, 2, 1, 3))
        ol = torch.empty((B, T, H, d), dtype=torch.float16, device=dev)
        S = self.SPLIT_K if (N >= 8192 and Np % (64 * self.SPLIT_K) == 0) else 1
        if S > 1:   # K = Np in S slices as a batch dimension (16 output tiles would leave most SMs idle), fp32 partials, one reduction
            ch = Np // S
            part = torch.empty((B * H, S, T, d), dtype=torch.float32, device=dev)
            ops.gemm(Pl.view(B * H, T, S, ch).permute(0, 2, 1, 3), vvT.view(B * H, d, S, ch).permute(0, 2, 1, 3), out=part)
            ops.sum_splits_cast(part.view(B, H, S, T, d), ol.permute(0, 2, 1, 3))
        else:
            ops.gemm(Pl, vvT.view(B, H, d, Np), out=ol.permute(0, 2, 1, 3))
        return ov, ol

    def _finish(self, ov, ol, v_epilogue, l_epilogue, B, N, T, Cv):
        E = self.embed_dim
        ve = v_epilogue or {}
        le = l_epilogue or {}
        dv = ops.gemm(ov.view(B * N, E), w16(self.out_v_proj.weight), bias=f32(self.out_v_proj.bias),
                      out_dtype=ve.get("out_dtype", torch.float16), gate=ve.get("gate"), gate_mode=VEC_PER_COL if ve else 0,
                      residual=ve["residual"].view(B * N, Cv) if ve else None)
        dl = ops.gemm(ol.view(B * T, E), w16(self.out_l_proj.weight), bias=f32(self.out_l_proj.bias),
                      out_dtype=torch.float32, gate=le.get("gate"), gate_mode=VEC_PER_COL if le else 0,
                      residual=le["residual"].view(B * T, -1) if le else None)
        return dv.view(B, N, Cv), dl.view(B, T, -1)

    @torch.no_grad()
    def forward(self, v, l, attention_mask_l=None):
        """Reference signature (:218): v [B,N,v_dim], l [B,T,l_dim] -> (attn_output_v, attn_output_l) in fp32."""
        if not v.is_cuda:
            raise MqdetError("BiMultiHeadAttention: CUDA tensors required (no CPU fallback)")
        dv, dl = self._attend(ops.cast_f16(v.contiguous()), ops.cast_f16(l.contiguous()), attention_mask_l)
        return ops.cast_f32(dv), dl


class BiAttentionBlockForCheckpoint(nn.Module):
    def __init__(self, v_dim, l_dim, embed_dim, num_heads, hidden_dim=None, dropout=0.1, drop_path=.0, init_values=1e-4,
                 cfg=None):
        super().__init__()
        self.layer_norm_v = nn.LayerNorm(v_dim)
        self.layer_norm_l = nn.LayerNorm(l_dim)
        self.attn = BiMultiHeadAttention(v_dim=v_dim, l_dim=l_dim, embed_dim=embed_dim, num_heads=num_heads,
                                         dropout=dropout, cfg=cfg)
        self.drop_path = nn.Identity()  # eval
        self.gamma_v = nn.Parameter(init_values * torch.ones((v_dim)), requires_grad=True)
        self.gamma_l = nn.Parameter(init_values * torch.ones((l_dim)), requires_grad=True)
        self.cfg = cfg
        if cfg.MODEL.DYHEAD.FUSE_CONFIG.SEPARATE_BIDIRECTIONAL:
            raise NotImplementedError("SEPARATE_BIDIRECTIONAL is False in every MQ-GLIP config")

    @torch.no_grad()
    def forward_flat(self, v16, l32, attention_mask_l):
        """Tower fast path: v16 [B,N,256] fp16 (levels concatenated), l32 [B,T,768] fp32 -> (v' fp16, l' fp32)."""
        nv, nl = self.layer_norm_v, self.layer_norm_l
        vn16 = ops.layernorm(v16, f32(nv.weight), f32(nv.bias), nv.eps)
        ln16, ln32 = ops.layernorm(l32, f32(nl.weight), f32(nl.bias), nl.eps, out16=True, out32=True)
        # v' = LN(v) + gamma_v * dv ; l' = LN(l) + gamma_l * dl   (residual on the normalised inputs, :420-425)
        return self.attn._attend(vn16, ln16, attention_mask_l,
                                 v_epilogue=dict(gate=f32(self.gamma_v), residual=vn16),
                                 l_epilogue=dict(gate=f32(self.gamma_l), residual=ln32))

    @torch.no_grad()
    def forward_flat_split(self, v16, l32, attention_mask_l):
        """forward_flat in two halves for two-stream execution: returns (v' fp16, ctx) after the image side; ``finish_text(ctx)``
        -> l' fp32 runs the text side (it depends on nothing the visual branch computes afterwards).  None when the product
        path does not apply (score_precision "f32", unusual shapes)."""
        a = self.attn
        B, N, Cv = v16.shape
        if not a._fused_applies(Cv, l32.shape[1]):
            return None
        nv, nl = self.layer_norm_v, self.layer_norm_l
        vn16 = ops.layernorm(v16, f32(nv.weight), f32(nv.bias), nv.eps)
        ln16, ln32 = ops.layernorm(l32, f32(nl.weight), f32(nl.bias), nl.eps, out16=True, out32=True)
        dv, ctx = a._fused_image(vn16, ln16, attention_mask_l, dict(gate=f32(self.gamma_v), residual=vn16))
        ctx["ln32"] = ln32
        return dv.view(B, N, Cv), ctx

    @torch.no_grad()
    def finish_text(self, ctx):
        return self.attn._fused_text(ctx, dict(gate=f32(self.gamma_l), residual=ctx["ln32"]))

    def single_attention_call(self, v, l, attention_mask_l=None, dummy_tensor=None):
        v2, l2 = self.forward_flat(ops.cast_f16(v.contiguous()), l.float().contiguous(), attention_mask_l)
        return ops.cast_f32(v2), l2

    @torch.no_grad()
    def forward(self, q0, q1, q2, q3, q4, l, attention_mask_l=None, dummy_tensor=None):
        """Reference signature (:377): five [B,256,h,w] maps + l -> 10-tuple (5 maps, new l, 4 x None)."""
        feats = [q0, q1, q2, q3, q4]
        if not q0.is_cuda:
            raise MqdetError("BiAttentionBlockForCheckpoint: CUDA tensors required (no CPU fallback)")
        sizes = [(f.shape[2], f.shape[3]) for f in feats]
        v = _flatten_levels(feats)
        new_v, new_l = self.single_attention_call(v, l, attention_mask_l)
        lv = _split_levels(new_v, sizes)
        return lv[0], lv[1], lv[2], lv[3], lv[4], new_l, None, None, None, None
