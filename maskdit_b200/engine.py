"""Forward / backward orchestration of the MaskDiT network over the sm_90a kernels.

This is the arithmetic of `DiT.forward` + `forward_encoder` (models/maskdit.py:467-557) and of its autograd
backward, expressed as a fixed sequence of C-ABI kernel launches on the current CUDA stream:

  forward  (per DiTBlock, models/maskdit.py:188-192)
      LN+modulate -> qkv GEMM -> attention -> proj GEMM (+bias, *gate, +residual fused)
      LN+modulate -> fc1 GEMM (+bias, GELU fused) -> fc2 GEMM (+bias, *gate, +residual fused)
  backward (hand-written; the reference gets it from autograd)
      gate-bwd -> dgrad GEMM (GELU' fused) / wgrad GEMM (stream-K) -> LN-modulate-bwd -> attention-bwd ...

Residual stream, LayerNorm statistics, softmax, modulation vectors, loss and all gradients w.r.t. parameters are
fp32; GEMM operands are bf16 with fp32 accumulation in registers.  Nothing here falls back to PyTorch math.
"""
from __future__ import annotations

import ctypes

import torch

from . import ops
from .ops import EPI_ATOMIC, EPI_DGELU, EPI_GATE_RESID, EPI_GELU, EPI_STORE, bf16, f32, gemm


class BlockSpec:
    """Static description of one DiTBlock's place in the parameter set / modulation vector."""

    def __init__(self, prefix, dim, heads, mod_off):
        self.prefix, self.dim, self.heads, self.mod_off = prefix, dim, heads, mod_off
        self.dh = dim // heads


class Engine:
    """Kernel-by-kernel reference of the step driver's launch sequence, for the default mode only: under
    `mdt_set_deterministic(1)` the per-kernel entry points it calls for the patch-embedding, mask-token and fused
    LN/gate bias gradients need scratch and return MDT_ERR_UNSUPPORTED (raised here), since only the step driver
    (`CEngine`) carries that scratch in its workspace."""

    def __init__(self, cfg, store):
        self.cfg, self.store = cfg, store
        # dec_hidden == 0: the decoder-less DiT (use_decoder=False), final layer on the encoder width
        self.has_dec = cfg.dec_hidden > 0
        o0, self.NA, hidden = store.ada_w_range

        def mod_off(prefix):
            """Column of the head's modulation vector: the first row of its adaLN weight in the [NA, hidden] matrix."""
            return (store.offsets[f"{prefix}.adaLN_modulation.1.weight"][0] - o0) // hidden

        self.enc = [BlockSpec(p, cfg.hidden, cfg.heads, mod_off(p))
                    for p in (f"model.blocks.{i}" for i in range(cfg.depth))]
        self.dec = [BlockSpec(p, cfg.dec_hidden, cfg.dec_heads, mod_off(p))
                    for p in (f"model.decoder_blocks.{i}" for i in range(cfg.dec_depth))]
        self.off_declayer = mod_off("model.decoder_layer") if self.has_dec else None
        self.off_final = mod_off("model.final_layer")

    # ------------------------------------------------------------------------------------------------------
    def w16(self, key):
        return self.store.view16(key)

    def w32(self, key):
        return self.store.view32(key)

    def _ada_all(self):
        o, rows, hid = self.store.ada_w_range
        ob, _ = self.store.ada_b_range
        return self.store.w16[o:o + rows * hid], self.store.w32[ob:ob + rows]

    def _label_operands(self, labels):
        """bf16 one-hot/soft labels [B, Kp] and label table [D, Kp]; Kp = num_classes padded to 8 for TMA strides."""
        nc = self.cfg.num_classes
        y16 = ops.cast_bf16(labels.contiguous())
        Wy = self.w16("model.y_embedder.embedding_table.weight")
        if nc % 8 == 0:
            return y16, Wy, nc
        Kp = (nc + 7) // 8 * 8  # only for toy class counts; the registry configs use 1000
        return (torch.nn.functional.pad(y16, (0, Kp - nc)).contiguous(),
                torch.nn.functional.pad(Wy, (0, Kp - nc)).contiguous(), Kp)

    # ------------------------------------------------------------------------------------------------------
    def forward(self, x_in, sigma, labels, mask_dict, save):
        """x_in [B,C,R,R] f32 (UNscaled network input; c_in is applied inside), sigma [B] f32, labels [B,nc] f32
        or None, mask_dict {'ids_keep','ids_restore','mask'} or None (= no token dropping).
        Returns (F [B*L, p*p*C] f32, ctx or None)."""
        cfg = self.cfg
        B = x_in.shape[0]
        D, Dd, L, p = cfg.hidden, cfg.dec_hidden, cfg.num_patches, cfg.patch
        ids_keep = mask_dict["ids_keep"] if mask_dict is not None else None
        ids_restore = mask_dict["ids_restore"] if mask_dict is not None else None
        T = ids_keep.shape[1] if ids_keep is not None else L
        Me, Md, NA = B * T, B * L, self.NA
        ctx = {} if save else None

        X = ops.patch_embed(x_in, sigma, cfg.sigma_data, self.w32("model.x_embedder.proj.weight").view(D, -1),
                            self.w32("model.x_embedder.proj.bias"), self.w32("model.pos_embed").view(L, D),
                            ids_keep, p, D).view(Me, D)
        # conditioning: c = t_emb(c_noise) + y_emb(labels)   (models/maskdit.py:491-495, :767)
        tf = ops.timestep_freq(sigma, 256)
        th_pre = torch.empty(B, D, dtype=f32, device=X.device)
        gemm(tf, self.w16("model.t_embedder.mlp.0.weight"), B, D, 256, out=th_pre,
             bias=self.w32("model.t_embedder.mlp.0.bias"))
        th = ops.silu(th_pre)
        c = torch.empty(B, D, dtype=f32, device=X.device)
        gemm(th, self.w16("model.t_embedder.mlp.2.weight"), B, D, D, out=c,
             bias=self.w32("model.t_embedder.mlp.2.bias"))
        y16 = None
        if cfg.num_classes:
            y16, Wy, Kp = self._label_operands(labels)
            c2 = torch.empty_like(c)
            gemm(y16, Wy, B, D, Kp, out=c2, resid=c, ld_resid=D)
            c = c2
        sc = ops.silu(c)
        Wada, bada = self._ada_all()
        mod = torch.empty(B, NA, dtype=f32, device=X.device)
        gemm(sc, Wada, B, NA, D, out=mod, bias=bada)
        if save:
            ctx.update(x_in=x_in, sigma=sigma, ids_keep=ids_keep, ids_restore=ids_restore, tf=tf, th_pre=th_pre,
                       th=th, c=c, sc=sc, y16=y16, mod=mod, B=B, T=T, enc=[], dec=[])

        for spec in self.enc:
            X, saved = self._block_fwd(spec, X, mod, B, T, save)
            if save:
                ctx["enc"].append(saved)

        pd = cfg.patch_dim
        if not self.has_dec:
            # FinalLayer on the encoder's tokens (models/maskdit.py:550); with a mask the kept rows are scattered back
            # and the removed ones are zeros (:551-553)
            o = self.off_final
            xf, mean_f, rstd_f = ops.ln_modulate(X, mod[:, o:], mod[:, o + D:], NA, T, Me, D, save_stats=save)
            Fk = torch.empty(Me, pd, dtype=f32, device=X.device)
            gemm(xf, self.w16("model.final_layer.linear.weight"), Me, pd, D, out=Fk,
                 bias=self.w32("model.final_layer.linear.bias"))
            Fo = Fk if ids_restore is None else ops.unmask_tokens(Fk, None, None, ids_restore, B, T, L, pd).view(Md, pd)
            if save:
                ctx.update(X_enc=X, xf=xf, mean_f=mean_f, rstd_f=rstd_f)
            return Fo, ctx

        # DecoderLayer (models/maskdit.py:209-213) + unmask_tokens + decoder_pos_embed (:539-545)
        o = self.off_declayer
        xmd, mean_d, rstd_d = ops.ln_modulate(X, mod[:, o:], mod[:, o + D:], NA, T, Me, D, save_stats=save)
        u = torch.empty(Me, Dd, dtype=f32, device=X.device)
        gemm(xmd, self.w16("model.decoder_layer.linear.weight"), Me, Dd, D, out=u,
             bias=self.w32("model.decoder_layer.linear.bias"))
        tok = self.w32("model.mask_token").view(Dd) if "model.mask_token" in self.store.offsets else None
        Z = ops.unmask_tokens(u, tok, self.w32("model.decoder_pos_embed").view(L, Dd), ids_restore, B, T, L,
                              Dd).view(Md, Dd)
        if save:
            ctx.update(X_enc=X, xmd=xmd, mean_d=mean_d, rstd_d=rstd_d)
        for spec in self.dec:
            Z, saved = self._block_fwd(spec, Z, mod, B, L, save)
            if save:
                ctx["dec"].append(saved)
        # FinalLayer (models/maskdit.py:230-234)
        o = self.off_final
        xf, mean_f, rstd_f = ops.ln_modulate(Z, mod[:, o:], mod[:, o + Dd:], NA, L, Md, Dd, save_stats=save)
        Fo = torch.empty(Md, pd, dtype=f32, device=X.device)
        gemm(xf, self.w16("model.final_layer.linear.weight"), Md, pd, Dd, out=Fo,
             bias=self.w32("model.final_layer.linear.bias"))
        if save:
            ctx.update(Z_out=Z, xf=xf, mean_f=mean_f, rstd_f=rstd_f)
        return Fo, ctx

    def _block_fwd(self, s: BlockSpec, X, mod, B, T, save):
        """DiTBlock.forward (models/maskdit.py:188-192).  X [M, D] f32 -> X2 [M, D] f32."""
        D, M, NA, o, p = s.dim, B * T, self.NA, s.mod_off, s.prefix
        dev = X.device
        xm1, mean1, rstd1 = ops.ln_modulate(X, mod[:, o:], mod[:, o + D:], NA, T, M, D, save_stats=save)
        qkv = torch.empty(M, 3 * D, dtype=bf16, device=dev)
        gemm(xm1, self.w16(f"{p}.attn.qkv.weight"), M, 3 * D, D, out=qkv, bias=self.w32(f"{p}.attn.qkv.bias"))
        O, lse = ops.attention_fwd(qkv, B, T, s.heads, s.dh, need_lse=save)
        X1 = torch.empty(M, D, dtype=f32, device=dev) if save else X
        y1 = torch.empty(M, D, dtype=bf16, device=dev) if save else None
        gemm(O, self.w16(f"{p}.attn.proj.weight"), M, D, D, out=X1, bias=self.w32(f"{p}.attn.proj.bias"),
             epi=EPI_GATE_RESID, aux=y1, ld_aux=D, resid=X, ld_resid=D, gate=mod[:, o + 2 * D:], ld_gate=NA,
             rows_per_group=T)
        xm2, mean2, rstd2 = ops.ln_modulate(X1, mod[:, o + 3 * D:], mod[:, o + 4 * D:], NA, T, M, D, save_stats=save)
        H4 = self.store.offsets[f"{p}.mlp.fc1.weight"][2][0]
        a = torch.empty(M, H4, dtype=bf16, device=dev)
        hpre = torch.empty(M, H4, dtype=bf16, device=dev) if save else None
        gemm(xm2, self.w16(f"{p}.mlp.fc1.weight"), M, H4, D, out=a, bias=self.w32(f"{p}.mlp.fc1.bias"), epi=EPI_GELU,
             aux=hpre, ld_aux=H4)
        X2 = torch.empty(M, D, dtype=f32, device=dev) if save else X1
        y2 = torch.empty(M, D, dtype=bf16, device=dev) if save else None
        gemm(a, self.w16(f"{p}.mlp.fc2.weight"), M, D, H4, out=X2, bias=self.w32(f"{p}.mlp.fc2.bias"),
             epi=EPI_GATE_RESID, aux=y2, ld_aux=D, resid=X1, ld_resid=D, gate=mod[:, o + 5 * D:], ld_gate=NA,
             rows_per_group=T)
        saved = None
        if save:
            saved = dict(X=X, mean1=mean1, rstd1=rstd1, xm1=xm1, qkv=qkv, O=O, lse=lse, y1=y1, X1=X1, mean2=mean2,
                         rstd2=rstd2, xm2=xm2, hpre=hpre, a=a, y2=y2)
        return X2, saved

    # ------------------------------------------------------------------------------------------------------
    def backward(self, ctx, dF16):
        """Accumulate d(loss)/d(params) into the flat gradient buffer given dF [B*L, pd] bf16."""
        cfg, st = self.cfg, self.store
        st.ensure_grad()
        G = st.gview
        B, T = ctx["B"], ctx["T"]
        D, Dd, L, p, pd = cfg.hidden, cfg.dec_hidden, cfg.num_patches, cfg.patch, cfg.patch_dim
        Me, Md, NA = B * T, B * L, self.NA
        mod = ctx["mod"]
        dev = mod.device
        dmod = torch.zeros(B, NA, dtype=f32, device=dev)

        # the LN backward that starts the encoder's residual-stream gradient: of the decoder layer, or of the final
        # layer when there is no decoder
        o = self.off_final
        if not self.has_dec:
            # ---- final layer on the kept tokens: the removed tokens' rows are constant zeros in the forward
            # (models/maskdit.py:551-553), so their dF (the MAE term's gradient seed) is dropped
            dFk = dF16 if ctx["ids_keep"] is None else ops.gather_rows_bf16(dF16, ctx["ids_keep"], B, T, L, pd)
            self._wgrad(dFk, ctx["xf"], pd, D, Me, G("model.final_layer.linear.weight"))
            ops.colsum(dFk, G("model.final_layer.linear.bias"))
            dx_top = torch.empty(Me, D, dtype=bf16, device=dev)
            gemm(dFk, self.w16("model.final_layer.linear.weight"), Me, D, pd, b_mn=True, out=dx_top)
            del dFk
            mean_top, rstd_top = ctx["mean_f"], ctx["rstd_f"]
        else:
            # ---- final layer
            self._wgrad(dF16, ctx["xf"], pd, Dd, Md, G("model.final_layer.linear.weight"))
            ops.colsum(dF16, G("model.final_layer.linear.bias"))
            dxf = torch.empty(Md, Dd, dtype=bf16, device=dev)
            gemm(dF16, self.w16("model.final_layer.linear.weight"), Md, Dd, pd, b_mn=True, out=dxf)
            Gz = torch.empty(Md, Dd, dtype=f32, device=dev)
            # every LN backward finishes the residual-stream gradient that the NEXT gate backward consumes: one fused
            # pass
            dec, dec_sv = list(reversed(self.dec)), list(reversed(ctx["dec"]))
            dy2 = ops.ln_modulate_bwd_gate(dxf, ctx["Z_out"], ctx["mean_f"], ctx["rstd_f"], mod[:, o + Dd:], NA, L, Gz,
                                           False, dmod[:, o:], dmod[:, o + Dd:], NA, Md, Dd,
                                           gate_next=self._mlp_gate(dec[0], dec_sv[0], mod, dmod) if dec else None)
            # ---- decoder blocks
            for i, (spec, saved) in enumerate(zip(dec, dec_sv)):
                nxt = self._mlp_gate(dec[i + 1], dec_sv[i + 1], mod, dmod) if i + 1 < len(dec) else None
                dy2 = self._block_bwd(spec, saved, Gz, mod, dmod, B, L, dy2, nxt)
            # ---- unmask + decoder layer
            tok_g = G("model.mask_token").view(Dd) if "model.mask_token" in st.offsets and \
                ctx["ids_restore"] is not None else None
            du = ops.unmask_tokens_bwd(Gz, ctx["ids_restore"], tok_g, B, T, L, Dd)
            del Gz
            o = self.off_declayer
            self._wgrad(du, ctx["xmd"], Dd, D, Me, G("model.decoder_layer.linear.weight"))
            ops.colsum(du, G("model.decoder_layer.linear.bias"))
            dx_top = torch.empty(Me, D, dtype=bf16, device=dev)
            gemm(du, self.w16("model.decoder_layer.linear.weight"), Me, D, Dd, b_mn=True, out=dx_top)
            mean_top, rstd_top = ctx["mean_d"], ctx["rstd_d"]
        Ge = torch.empty(Me, D, dtype=f32, device=dev)
        enc, enc_sv = list(reversed(self.enc)), list(reversed(ctx["enc"]))
        dy2 = ops.ln_modulate_bwd_gate(dx_top, ctx["X_enc"], mean_top, rstd_top, mod[:, o + D:], NA, T, Ge,
                                       False, dmod[:, o:], dmod[:, o + D:], NA, Me, D,
                                       gate_next=self._mlp_gate(enc[0], enc_sv[0], mod, dmod) if enc else None)
        del dx_top
        # ---- encoder blocks
        for i, (spec, saved) in enumerate(zip(enc, enc_sv)):
            nxt = self._mlp_gate(enc[i + 1], enc_sv[i + 1], mod, dmod) if i + 1 < len(enc) else None
            dy2 = self._block_bwd(spec, saved, Ge, mod, dmod, B, T, dy2, nxt)
        # ---- patch embedding (no input gradient needed)
        ops.patch_embed_bwd(ctx["x_in"], ctx["sigma"], cfg.sigma_data, ctx["ids_keep"], Ge.view(B, T, D),
                            G("model.x_embedder.proj.weight").view(D, -1), G("model.x_embedder.proj.bias"), p)
        del Ge
        # ---- adaLN projections of all blocks at once, then the conditioning MLPs
        dmod16 = ops.cast_bf16(dmod)
        ow, rows, hid = st.ada_w_range
        ob, _ = st.ada_b_range
        gW = st.grad[ow:ow + rows * hid]
        self._wgrad(dmod16, ctx["sc"], NA, D, B, gW)
        ops.colsum(dmod, st.grad[ob:ob + rows])
        dsc = torch.zeros(B, D, dtype=f32, device=dev)
        Wada, _ = self._ada_all()
        gemm(dmod16, Wada, B, D, NA, b_mn=True, out=dsc, epi=EPI_ATOMIC)  # K = NA is long: stream-K
        dc32, dc16 = ops.silu_bwd(dsc, ctx["c"])
        if cfg.num_classes:
            nc = cfg.num_classes
            y16 = ctx["y16"]
            if nc % 8 == 0:
                self._wgrad(dc16, y16, D, nc, B, G("model.y_embedder.embedding_table.weight"))
            else:
                Kp = y16.shape[1]
                tmp = torch.zeros(D, Kp, dtype=f32, device=dev)
                self._wgrad(dc16, y16, D, Kp, B, tmp)
                G("model.y_embedder.embedding_table.weight").add_(tmp[:, :nc])
        self._wgrad(dc16, ctx["th"], D, D, B, G("model.t_embedder.mlp.2.weight"))
        ops.colsum(dc32, G("model.t_embedder.mlp.2.bias"))
        dth = torch.zeros(B, D, dtype=f32, device=dev)
        gemm(dc16, self.w16("model.t_embedder.mlp.2.weight"), B, D, D, b_mn=True, out=dth, epi=EPI_ATOMIC)
        dpre32, dpre16 = ops.silu_bwd(dth, ctx["th_pre"])
        self._wgrad(dpre16, ctx["tf"], D, 256, B, G("model.t_embedder.mlp.0.weight"))
        ops.colsum(dpre32, G("model.t_embedder.mlp.0.bias"))

    def _wgrad(self, dY, Xin, n_out, k_in, tokens, gout):
        """gout[n_out, k_in] += dY[tokens, n_out]^T @ Xin[tokens, k_in]   (stream-K, fp32 red.add)"""
        gemm(dY, Xin, n_out, k_in, tokens, a_mn=True, b_mn=True, out=gout, ldo=k_in, epi=EPI_ATOMIC)

    def _mlp_gate(self, s: BlockSpec, sv, mod, dmod):
        """Arguments of the MLP-branch gate backward of block `s` (consumed by ops.ln_modulate_bwd_gate)."""
        o, D = s.mod_off, s.dim
        return (sv["y2"], mod[:, o + 5 * D:], self.NA, dmod[:, o + 5 * D:], self.NA,
                self.store.gview(f"{s.prefix}.mlp.fc2.bias"))

    def _block_bwd(self, s: BlockSpec, sv, Gr, mod, dmod, B, T, dy2=None, gate_next=None):
        """Backward of one DiTBlock; Gr [M, D] f32 is the residual-stream gradient, updated in place.
        `dy2` = gradient of this block's MLP-branch output when the caller's LN backward already produced it (fused
        gate backward); `gate_next` = the MLP gate of the block processed next, fused into this block's last LN
        backward, whose dy is returned."""
        D, M, NA, o, p = s.dim, B * T, self.NA, s.mod_off, s.prefix
        G = self.store.gview
        dev = Gr.device
        H4 = sv["a"].shape[1]
        # x2 = x1 + gate_mlp * (fc2(gelu(fc1(xm2))))
        if dy2 is None:
            dy2 = ops.gate_bwd(Gr, sv["y2"], mod[:, o + 5 * D:], NA, T, dmod[:, o + 5 * D:], NA,
                               G(f"{p}.mlp.fc2.bias"), M, D)
        dh = torch.empty(M, H4, dtype=bf16, device=dev)
        # the fc1 bias gradient (column sums of dh) is accumulated by the same epilogue that writes dh
        gemm(dy2, self.w16(f"{p}.mlp.fc2.weight"), M, H4, D, b_mn=True, out=dh, epi=EPI_DGELU, aux=sv["hpre"],
             ld_aux=H4, colsum=G(f"{p}.mlp.fc1.bias"))
        self._wgrad(dy2, sv["a"], D, H4, M, G(f"{p}.mlp.fc2.weight"))
        del dy2
        dxm2 = torch.empty(M, D, dtype=bf16, device=dev)
        gemm(dh, self.w16(f"{p}.mlp.fc1.weight"), M, D, H4, b_mn=True, out=dxm2)
        self._wgrad(dh, sv["xm2"], H4, D, M, G(f"{p}.mlp.fc1.weight"))
        del dh
        # x1 = x + gate_msa * proj(attn(qkv(xm1))): its gate backward rides on the LN2 backward
        dy1 = ops.ln_modulate_bwd_gate(dxm2, sv["X1"], sv["mean2"], sv["rstd2"], mod[:, o + 4 * D:], NA, T, Gr, True,
                                       dmod[:, o + 3 * D:], dmod[:, o + 4 * D:], NA, M, D,
                                       gate_next=(sv["y1"], mod[:, o + 2 * D:], NA, dmod[:, o + 2 * D:], NA,
                                                  G(f"{p}.attn.proj.bias")))
        dO = torch.empty(M, D, dtype=bf16, device=dev)
        gemm(dy1, self.w16(f"{p}.attn.proj.weight"), M, D, D, b_mn=True, out=dO)
        self._wgrad(dy1, sv["O"], D, D, M, G(f"{p}.attn.proj.weight"))
        del dy1
        dqkv = ops.attention_bwd(sv["qkv"], sv["O"], dO, sv["lse"], B, T, s.heads, s.dh)
        ops.colsum(dqkv, G(f"{p}.attn.qkv.bias"))
        dxm1 = torch.empty(M, D, dtype=bf16, device=dev)
        gemm(dqkv, self.w16(f"{p}.attn.qkv.weight"), M, D, 3 * D, b_mn=True, out=dxm1)
        self._wgrad(dqkv, sv["xm1"], 3 * D, D, M, G(f"{p}.attn.qkv.weight"))
        return ops.ln_modulate_bwd_gate(dxm1, sv["X"], sv["mean1"], sv["rstd1"], mod[:, o + D:], NA, T, Gr, True,
                                        dmod[:, o:], dmod[:, o + D:], NA, M, D, gate_next=gate_next)


RECOMPUTE_MARGIN = 256 << 20   # bytes kept free when the recompute count is chosen from the memory left


def pick_recompute(sizes, budget):
    """The smallest recompute count r whose training workspace `sizes[r]` (bytes, r = 0 .. depth + dec_depth) fits into
    `budget` bytes.  Raises torch.OutOfMemoryError naming the smallest workspace and the budget when none fits."""
    for r, n in enumerate(sizes):
        if n <= budget:
            return r
    r = min(range(len(sizes)), key=lambda i: sizes[i])
    raise torch.OutOfMemoryError(
        f"the training workspace does not fit: it needs {sizes[r] / 2**30:.2f} GiB even with {r} of "
        f"{len(sizes) - 1} blocks recomputed, and {max(budget, 0) / 2**30:.2f} GiB of device memory is available")


class CEngine:
    """The same forward / backward issued by the C++ step driver (csrc/driver.cu: `mdt_forward`, `mdt_backward`): ONE
    C-ABI call each over the packed parameter blob and one workspace buffer, instead of ~780 ctypes calls and a
    `torch.empty` per activation (70 ms of host time per step in round 1, which bound the 128-samples-per-GPU config).
    `Engine` above issues the identical launch sequence kernel by kernel and is kept as the cross-check
    (tests/test_model_gpu.py::check_c_driver_matches_engine).

    The C model handle it creates from the network's config is the one place the packed parameter layout is decided:
    the `FlatStore` of the module is built from it (`tensors`, `param_count`, `NA`) and assigned to `store`."""

    def __init__(self, cfg):
        self.cfg, self.store = cfg, None
        L = ops.lib()
        mc = ops.L.ModelCfg(cfg.img_resolution, cfg.img_channels, cfg.patch, cfg.num_classes, cfg.hidden, cfg.depth,
                            cfg.heads, cfg.mlp_hidden, cfg.dec_hidden, cfg.dec_depth, cfg.dec_heads, cfg.dec_mlp_hidden,
                            int(cfg.has_mask_token), cfg.sigma_data)
        h = ctypes.c_void_p()
        ops.check(L.mdt_model_create(ctypes.byref(mc), ctypes.byref(h)), "mdt_model_create", 0)
        self._h, self._L = h, L
        if getattr(cfg, "logvar_channels", 0):   # the learned loss weighting's tensors join the layout
            ops.check(L.mdt_model_set_logvar(h, cfg.logvar_channels), "mdt_model_set_logvar", 0)
        if getattr(cfg, "precond", 0):   # flow: sigma carries t, c_in = 1, c_noise = t
            ops.check(L.mdt_model_set_precond(h, cfg.precond), "mdt_model_set_precond", 0)
        self.NA = L.mdt_model_mod_width(h)   # width of the modulation vector = rows of the adaLN weight matrix
        # Activation recomputation (`mdt_model_set_recompute`) of the training pass.  `recompute` None: automatic, i.e.
        # nothing is recomputed unless the workspace allocation runs out of memory, then the smallest count that fits
        # (remembered per batch shape); an int forces that count.  `recompute_blocks`: the count of the last training
        # forward.
        self.recompute = None
        self.recompute_blocks = 0
        self._auto_recompute = {}

    def __del__(self):
        try:
            self._L.mdt_model_destroy(self._h)
        except Exception:
            pass

    def tensors(self):
        """{name: (offset, numel)} of every packed tensor, in blob order (`mdt_model_param_info`)."""
        name, off, num = ctypes.create_string_buffer(160), ctypes.c_longlong(), ctypes.c_longlong()
        out = {}
        for i in range(self._L.mdt_model_num_tensors(self._h)):
            ops.check(self._L.mdt_model_param_info(self._h, i, name, 160, ctypes.byref(off), ctypes.byref(num)),
                      "mdt_model_param_info", 0)
            out[name.value.decode()] = (off.value, num.value)
        return out

    def param_count(self, trainable_only):
        """Elements of the trainable region, or of the whole blob (`mdt_model_param_count`)."""
        return self._L.mdt_model_param_count(self._h, int(trainable_only))

    def fp32_read_ranges(self):
        """[(lo, hi)] of the trainable region that the training step reads from the fp32 masters
        (`mdt_model_fp32_read_ranges`)."""
        k = self._L.mdt_model_fp32_read_ranges(self._h, None, 0)
        ops.check(min(k, 0), "mdt_model_fp32_read_ranges", 0)
        buf = (ctypes.c_longlong * (2 * max(k, 1)))()
        ops.check(min(self._L.mdt_model_fp32_read_ranges(self._h, buf, k), 0), "mdt_model_fp32_read_ranges", 0)
        return [(buf[2 * i], buf[2 * i + 1]) for i in range(k)]

    @property
    def num_blocks(self):
        return self.cfg.depth + self.cfg.dec_depth

    def set_recompute(self, r):
        """Set the handle's recompute count (blocks 0 .. r-1 in forward order, encoder first)."""
        ops.check(self._L.mdt_model_set_recompute(self._h, int(r)), "mdt_model_set_recompute", 0)

    def workspace_bytes(self, B, T, training, recompute=None):
        """`mdt_workspace_bytes`; `recompute` (training only): at that count instead of the handle's current one."""
        cur = self._L.mdt_model_get_recompute(self._h)
        if recompute is not None:
            self.set_recompute(recompute)
        try:
            n = self._L.mdt_workspace_bytes(self._h, B, T, int(training))
        finally:
            if recompute is not None:
                self.set_recompute(cur)
        if n <= 0:
            raise ops.L.MdtError("mdt_workspace_bytes failed")
        return n

    def _count(self, masked, recompute=0):
        """Kernel launches of one forward / backward (for bench.py's gpu_launches claim): same sequence as `Engine`,
        plus the 7 forward launches of each recomputed block in the backward."""
        c = self.cfg
        nb = c.depth + c.dec_depth
        if c.dec_hidden == 0:   # no decoder: final 2 (+ zero-filled scatter) / final 4 (+ kept-row gather of dF)
            fwd = 9 + (2 if c.num_classes else 0) + 7 * nb + int(masked)          # embed/conditioning 7
            bwd = 16 + 13 * nb + (1 if c.num_classes else 0) + int(masked)        # patch-embed 1, conditioning 11
            return fwd, bwd + 7 * recompute
        fwd = 12 + (2 if c.num_classes else 0) + 7 * nb          # embed/conditioning 7, decoder layer 3, final 2
        bwd = 21 + 13 * nb + (1 if c.num_classes else 0)         # final 4, transition 5, patch-embed 1, conditioning 11
        return fwd, bwd + 7 * recompute

    def _training_workspace(self, B, T, device):
        """The recompute count and the workspace of a training pass.  Forced count: that plan.  Automatic: the count
        chosen earlier for this batch shape, else r = 0; only when that allocation runs out of memory, the smallest
        count whose workspace fits into the free device memory plus the caching allocator's reserved-but-unused bytes,
        less RECOMPUTE_MARGIN."""
        key = (B, T, self._L.mdt_get_deterministic())   # the deterministic mode's scratch is part of the workspace
        r =self.recompute if self.recompute is not None else self._auto_recompute.get(key, 0)
        self.set_recompute(r)
        nbytes = self.workspace_bytes(B, T, True)
        try:
            return r, torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes
        except torch.OutOfMemoryError:
            if self.recompute is not None or r > 0:
                raise
        free, _ = torch.cuda.mem_get_info(device)
        budget = free + torch.cuda.memory_reserved(device) - torch.cuda.memory_allocated(device) - RECOMPUTE_MARGIN
        r = pick_recompute([self.workspace_bytes(B, T, True, k) for k in range(self.num_blocks + 1)], budget)
        self._auto_recompute[key] = r
        self.set_recompute(r)
        nbytes = self.workspace_bytes(B, T, True)
        return r, torch.empty(nbytes, dtype=torch.uint8, device=device), nbytes

    def forward(self, x_in, sigma, labels, mask_dict, save):
        cfg = self.cfg
        B, L = x_in.shape[0], cfg.num_patches
        ids_keep = mask_dict["ids_keep"] if mask_dict is not None else None
        ids_restore = mask_dict["ids_restore"] if mask_dict is not None else None
        T = ids_keep.shape[1] if ids_keep is not None else L
        for t, dt in ((x_in, f32), (sigma, f32), (labels, f32), (ids_keep, torch.int64), (ids_restore, torch.int64)):
            ops._c(t, dt)
        ops.L.sync_deterministic()   # the workspace size and the backward's reductions follow the torch flag
        if save:   # ONE allocation per pass
            r, ws, nbytes = self._training_workspace(B, T, x_in.device)
            self.recompute_blocks = r
        else:
            nbytes = self.workspace_bytes(B, T, False)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x_in.device)
        Fo = torch.empty(B * L, cfg.patch_dim, dtype=f32, device=x_in.device)
        st = self.store
        ops.check(self._L.mdt_forward(self._h, ops.ptr(st.w32), ops.ptr(st.w16), ops.ptr(x_in), ops.ptr(sigma),
                                      ops.ptr(labels), ops.ptr(ids_keep), ops.ptr(ids_restore), B, T, int(save),
                                      ops.ptr(ws), nbytes, ops.ptr(Fo), ops.stream_ptr()), "mdt_forward",
                  self._count(ids_restore is not None)[0])
        ctx = None
        if save:
            ctx = dict(ws=ws, nbytes=nbytes, x_in=x_in, sigma=sigma, ids_keep=ids_keep, ids_restore=ids_restore, B=B,
                       T=T, recompute=r)
        return Fo, ctx

    def backward(self, ctx, dF16):
        st = self.store
        st.ensure_grad()
        ops._c(dF16, bf16)
        ops.L.sync_deterministic()
        self.set_recompute(ctx["recompute"])   # the plan the forward laid the workspace out with
        ops.check(self._L.mdt_backward(self._h, ops.ptr(st.w32), ops.ptr(st.w16), ops.ptr(st.grad), ops.ptr(ctx["x_in"]),
                                       ops.ptr(ctx["sigma"]), ops.ptr(ctx["ids_keep"]), ops.ptr(ctx["ids_restore"]),
                                       ops.ptr(dF16), ctx["B"], ctx["T"], ops.ptr(ctx["ws"]), ctx["nbytes"],
                                       ops.L.GRAD_READY_FN(), None, ops.stream_ptr()), "mdt_backward",
                  self._count(ctx["ids_restore"] is not None, ctx["recompute"])[1])
