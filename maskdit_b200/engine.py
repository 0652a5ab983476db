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

import torch

from . import ops
from .ops import EPI_ATOMIC, EPI_DGELU, EPI_GATE_RESID, EPI_GELU, EPI_STORE, bf16, f32, gemm


class BlockSpec:
    """Static description of one DiTBlock's place in the parameter set / modulation vector."""

    def __init__(self, prefix, dim, heads, mod_off):
        self.prefix, self.dim, self.heads, self.mod_off = prefix, dim, heads, mod_off
        self.dh = dim // heads


class Engine:
    def __init__(self, cfg, store):
        self.cfg, self.store = cfg, store
        D, Dd = cfg.hidden, cfg.dec_hidden
        off = 0
        self.enc = []
        for i in range(cfg.depth):
            self.enc.append(BlockSpec(f"model.blocks.{i}", D, cfg.heads, off))
            off += 6 * D
        self.off_declayer = off
        off += 2 * D
        self.dec = []
        for i in range(cfg.dec_depth):
            self.dec.append(BlockSpec(f"model.decoder_blocks.{i}", Dd, cfg.dec_heads, off))
            off += 6 * Dd
        self.off_final = off
        off += 2 * Dd
        self.NA = off
        assert store.ada_w_range[1] == self.NA, (store.ada_w_range, self.NA)

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
        pd = cfg.patch_dim
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
    def backward(self, ctx, dF16, on_ready=None):
        """Accumulate d(loss)/d(params) into the flat gradient buffer given dF [B*L, pd] bf16.
        `on_ready(lo, hi)` (optional) is called as soon as the gradient elements [lo, hi) are final, i.e. right after
        the kernels of a block's backward have been enqueued: the training step uses it to overlap the gradient
        all-reduce and the optimizer with the rest of the backward (what DDP buckets do in the reference)."""
        cfg, st = self.cfg, self.store
        st.ensure_grad()
        G = st.gview
        B, T = ctx["B"], ctx["T"]
        D, Dd, L, p, pd = cfg.hidden, cfg.dec_hidden, cfg.num_patches, cfg.patch, cfg.patch_dim
        Me, Md, NA = B * T, B * L, self.NA
        mod = ctx["mod"]
        dev = mod.device
        dmod = torch.zeros(B, NA, dtype=f32, device=dev)

        # ---- final layer
        o = self.off_final
        self._wgrad(dF16, ctx["xf"], pd, Dd, Md, G("model.final_layer.linear.weight"))
        ops.colsum(dF16, G("model.final_layer.linear.bias"))
        dxf = torch.empty(Md, Dd, dtype=bf16, device=dev)
        gemm(dF16, self.w16("model.final_layer.linear.weight"), Md, Dd, pd, b_mn=True, out=dxf)
        Gz = torch.empty(Md, Dd, dtype=f32, device=dev)
        # every LN backward finishes the residual-stream gradient that the NEXT gate backward consumes: one fused pass
        dec, dec_sv = list(reversed(self.dec)), list(reversed(ctx["dec"]))
        dy2 = ops.ln_modulate_bwd_gate(dxf, ctx["Z_out"], ctx["mean_f"], ctx["rstd_f"], mod[:, o + Dd:], NA, L, Gz,
                                       False, dmod[:, o:], dmod[:, o + Dd:], NA, Md, Dd,
                                       gate_next=self._mlp_gate(dec[0], dec_sv[0], mod, dmod) if dec else None)
        # ---- decoder blocks
        for i, (spec, saved) in enumerate(zip(dec, dec_sv)):
            nxt = self._mlp_gate(dec[i + 1], dec_sv[i + 1], mod, dmod) if i + 1 < len(dec) else None
            dy2 = self._block_bwd(spec, saved, Gz, mod, dmod, B, L, dy2, nxt)
            if on_ready is not None:
                on_ready(*st.prefix_range(spec.prefix + "."))
        # ---- unmask + decoder layer
        tok_g = G("model.mask_token").view(Dd) if "model.mask_token" in st.offsets and ctx["ids_restore"] is not None \
            else None
        du = ops.unmask_tokens_bwd(Gz, ctx["ids_restore"], tok_g, B, T, L, Dd)
        del Gz
        o = self.off_declayer
        self._wgrad(du, ctx["xmd"], Dd, D, Me, G("model.decoder_layer.linear.weight"))
        ops.colsum(du, G("model.decoder_layer.linear.bias"))
        dxmd = torch.empty(Me, D, dtype=bf16, device=dev)
        gemm(du, self.w16("model.decoder_layer.linear.weight"), Me, D, Dd, b_mn=True, out=dxmd)
        Ge = torch.empty(Me, D, dtype=f32, device=dev)
        enc, enc_sv = list(reversed(self.enc)), list(reversed(ctx["enc"]))
        dy2 = ops.ln_modulate_bwd_gate(dxmd, ctx["X_enc"], ctx["mean_d"], ctx["rstd_d"], mod[:, o + D:], NA, T, Ge,
                                       False, dmod[:, o:], dmod[:, o + D:], NA, Me, D,
                                       gate_next=self._mlp_gate(enc[0], enc_sv[0], mod, dmod) if enc else None)
        # ---- encoder blocks
        for i, (spec, saved) in enumerate(zip(enc, enc_sv)):
            nxt = self._mlp_gate(enc[i + 1], enc_sv[i + 1], mod, dmod) if i + 1 < len(enc) else None
            dy2 = self._block_bwd(spec, saved, Ge, mod, dmod, B, T, dy2, nxt)
            if on_ready is not None:
                on_ready(*st.prefix_range(spec.prefix + "."))
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


class CEngine:
    """The same forward / backward issued by the C++ step driver (csrc/driver.cu: `mdt_forward`, `mdt_backward`): ONE
    C-ABI call each over the packed parameter blob and one workspace buffer, instead of ~780 ctypes calls and a
    `torch.empty` per activation (70 ms of host time per step in round 1, which bound the 128-samples-per-GPU config).
    `Engine` above issues the identical launch sequence kernel by kernel and is kept as the cross-check
    (tests/test_model_gpu_extra.py::test_c_driver_matches_python_engine); MDT_ENGINE=py selects it."""

    def __init__(self, cfg, store):
        import ctypes
        self.cfg, self.store = cfg, store
        L = ops.lib()
        has_tok = "model.mask_token" in store.offsets
        h4e = store.offsets["model.blocks.0.mlp.fc1.weight"][2][0] if cfg.depth else 4 * cfg.hidden
        h4d = store.offsets["model.decoder_blocks.0.mlp.fc1.weight"][2][0] if cfg.dec_depth else 4 * cfg.dec_hidden
        R = int(round(cfg.num_patches ** 0.5)) * cfg.patch
        mc = ops.L.ModelCfg(R, cfg.img_channels, cfg.patch, cfg.num_classes, cfg.hidden, cfg.depth, cfg.heads, h4e,
                            cfg.dec_hidden, cfg.dec_depth, cfg.dec_heads, h4d, int(has_tok), cfg.sigma_data)
        h = ctypes.c_void_p()
        ops.check(L.mdt_model_create(ctypes.byref(mc), ctypes.byref(h)), "mdt_model_create", 0)
        self._h, self._L = h, L
        # the C driver's packed layout must be the store's: compare every tensor once
        n = L.mdt_model_num_tensors(h)
        if n != len(store.offsets):
            raise ops.L.MdtError(f"driver layout has {n} tensors, the module {len(store.offsets)}")
        name = ctypes.create_string_buffer(160)
        off, num = ctypes.c_longlong(), ctypes.c_longlong()
        for i in range(n):
            L.mdt_model_param_info(h, i, name, 160, ctypes.byref(off), ctypes.byref(num))
            k = name.value.decode()
            if k not in store.offsets or store.offsets[k][:2] != (off.value, num.value):
                raise ops.L.MdtError(f"driver layout mismatch at {k}: {store.offsets.get(k)} vs {(off.value, num.value)}")
        if L.mdt_model_param_count(h, 1) != store.n_train or L.mdt_model_param_count(h, 0) != store.n_total:
            raise ops.L.MdtError("driver blob length differs from the flat store")
        self.NA = L.mdt_model_mod_width(h)
        self.launches = {}

    def __del__(self):
        try:
            self._L.mdt_model_destroy(self._h)
        except Exception:
            pass

    def workspace_bytes(self, B, T, training):
        n = self._L.mdt_workspace_bytes(self._h, B, T, int(training))
        if n <= 0:
            raise ops.L.MdtError("mdt_workspace_bytes failed")
        return n

    def _count(self, save):
        """Kernel launches of one forward / backward (for bench.py's gpu_launches claim): same sequence as `Engine`."""
        c = self.cfg
        nb = c.depth + c.dec_depth
        fwd = 12 + (2 if c.num_classes else 0) + 7 * nb          # embed/conditioning 7, decoder layer 3, final 2
        bwd = 21 + 13 * nb + (1 if c.num_classes else 0)         # final 4, transition 5, patch-embed 1, conditioning 11
        return fwd, bwd

    def forward(self, x_in, sigma, labels, mask_dict, save):
        cfg = self.cfg
        B, L = x_in.shape[0], cfg.num_patches
        ids_keep = mask_dict["ids_keep"] if mask_dict is not None else None
        ids_restore = mask_dict["ids_restore"] if mask_dict is not None else None
        T = ids_keep.shape[1] if ids_keep is not None else L
        for t, dt in ((x_in, f32), (sigma, f32), (labels, f32), (ids_keep, torch.int64), (ids_restore, torch.int64)):
            ops._c(t, dt)
        nbytes = self.workspace_bytes(B, T, save)
        ws = torch.empty(nbytes, dtype=torch.uint8, device=x_in.device)   # ONE allocation per pass
        Fo = torch.empty(B * L, cfg.patch_dim, dtype=f32, device=x_in.device)
        st = self.store
        ops.check(self._L.mdt_forward(self._h, ops.ptr(st.w32), ops.ptr(st.w16), ops.ptr(x_in), ops.ptr(sigma),
                                      ops.ptr(labels), ops.ptr(ids_keep), ops.ptr(ids_restore), B, T, int(save),
                                      ops.ptr(ws), nbytes, ops.ptr(Fo), ops.stream_ptr()), "mdt_forward",
                  self._count(save)[0])
        ctx = None
        if save:
            ctx = dict(ws=ws, nbytes=nbytes, x_in=x_in, sigma=sigma, ids_keep=ids_keep, ids_restore=ids_restore, B=B,
                       T=T)
        return Fo, ctx

    def backward(self, ctx, dF16, on_ready=None):
        st = self.store
        st.ensure_grad()
        ops._c(dF16, bf16)
        cb = ops.L.GRAD_READY_FN(lambda user, lo, hi: on_ready(lo, hi)) if on_ready is not None \
            else ops.L.GRAD_READY_FN()
        ops.check(self._L.mdt_backward(self._h, ops.ptr(st.w32), ops.ptr(st.w16), ops.ptr(st.grad), ops.ptr(ctx["x_in"]),
                                       ops.ptr(ctx["sigma"]), ops.ptr(ctx["ids_keep"]), ops.ptr(ctx["ids_restore"]),
                                       ops.ptr(dF16), ctx["B"], ctx["T"], ops.ptr(ctx["ws"]), ctx["nbytes"], cb, None,
                                       ops.stream_ptr()), "mdt_backward", self._count(True)[1])


def make_engine(cfg, store):
    """MDT_ENGINE=py: kernel-by-kernel launches from Python (`Engine`); default: the C++ step driver (`CEngine`)."""
    import os
    return Engine(cfg, store) if os.environ.get("MDT_ENGINE", "c") == "py" else CEngine(cfg, store)
