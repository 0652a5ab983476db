"""Thin Python wrappers over the C ABI (one function per kernel entry point).  CUDA tensors only; no fallback."""
from __future__ import annotations

import torch

from . import _lib as L
from ._lib import (ACT_NONE, ACT_SILU, EPI_ATOMIC, EPI_DGELU, EPI_GATE_RESID, EPI_GELU, EPI_STORE, check, gemm, lib,
                   ptr, stream_ptr)

bf16, f32 = torch.bfloat16, torch.float32


def _c(t, dtype=None):
    if t is None:
        return None
    if not t.is_cuda:
        raise L.MdtError("maskdit_b200 kernels need CUDA tensors (no CPU fallback)")
    if dtype is not None and t.dtype != dtype:
        raise L.MdtError(f"expected {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise L.MdtError("expected a contiguous tensor")
    return t


def mask_indices(noise, len_keep):
    """get_mask for a given noise tensor (models/maskdit.py:88-113) -> dict like the reference's mask_dict."""
    _c(noise, f32)
    B, Lt = noise.shape
    ids_keep = torch.empty(B, len_keep, dtype=torch.int64, device=noise.device)
    ids_restore = torch.empty(B, Lt, dtype=torch.int64, device=noise.device)
    mask = torch.empty(B, Lt, dtype=f32, device=noise.device)
    check(lib().mdt_mask_indices(ptr(noise), B, Lt, len_keep, ptr(ids_keep), ptr(ids_restore), ptr(mask),
                                 stream_ptr()), "mdt_mask_indices")
    return {"mask": mask, "ids_keep": ids_keep, "ids_restore": ids_restore}


def patch_embed(x, sigma, sigma_data, W, bias, pos, ids_keep, p, D):
    _c(x, f32), _c(W, f32), _c(bias, f32), _c(pos, f32), _c(ids_keep, torch.int64), _c(sigma, f32)
    B, C, R, _ = x.shape
    T = ids_keep.shape[1] if ids_keep is not None else (R // p) ** 2
    out = torch.empty(B, T, D, dtype=f32, device=x.device)
    check(lib().mdt_patch_embed(ptr(x), ptr(sigma), sigma_data, ptr(W), ptr(bias), ptr(pos), ptr(ids_keep), ptr(out),
                                B, C, R, p, D, T, stream_ptr()), "mdt_patch_embed")
    return out


def patch_embed_bwd(x, sigma, sigma_data, ids_keep, g, gW, gb, p):
    _c(x, f32), _c(g, f32), _c(gW, f32), _c(gb, f32)
    B, C, R, _ = x.shape
    T, D = g.shape[1], g.shape[2]
    check(lib().mdt_patch_embed_bwd(ptr(x), ptr(sigma), sigma_data, ptr(ids_keep), ptr(g), ptr(gW), ptr(gb), B, C, R,
                                    p, D, T, stream_ptr()), "mdt_patch_embed_bwd")


def timestep_freq(sigma, dim=256):
    _c(sigma, f32)
    out = torch.empty(sigma.numel(), dim, dtype=bf16, device=sigma.device)
    check(lib().mdt_timestep_freq(ptr(sigma), sigma.numel(), dim, ptr(out), stream_ptr()), "mdt_timestep_freq")
    return out


def flow_timestep_freq(t, dim=256):
    """The timestep embedding's frequencies on c_noise = t (mdt_flow_timestep_freq)."""
    _c(t, f32)
    out = torch.empty(t.numel(), dim, dtype=bf16, device=t.device)
    check(lib().mdt_flow_timestep_freq(ptr(t), t.numel(), dim, ptr(out), stream_ptr()), "mdt_flow_timestep_freq")
    return out


def silu(a, b=None, want_sum=False):
    _c(a, f32), _c(b, f32)
    out = torch.empty(a.shape, dtype=bf16, device=a.device)
    s = torch.empty_like(a) if want_sum else None
    check(lib().mdt_silu(ptr(a), ptr(b), ptr(s), ptr(out), a.numel(), stream_ptr()), "mdt_silu")
    return (out, s) if want_sum else out


def silu_bwd(dy, x, want_f32=True, want_bf16=True):
    _c(dy, f32), _c(x, f32)
    d32 = torch.empty_like(x) if want_f32 else None
    d16 = torch.empty(x.shape, dtype=bf16, device=x.device) if want_bf16 else None
    check(lib().mdt_silu_bwd(ptr(dy), ptr(x), ptr(d32), ptr(d16), x.numel(), stream_ptr()), "mdt_silu_bwd")
    return d32, d16


def cast_bf16(x, out=None):
    _c(x, f32)
    if out is None:
        out = torch.empty(x.shape, dtype=bf16, device=x.device)
    check(lib().mdt_cast_f32_bf16(ptr(x), ptr(out), x.numel(), stream_ptr()), "mdt_cast_f32_bf16")
    return out


def colsum(x, out, M=None, N=None, ld=None):
    """out[N] += sum_m x[m, n]"""
    M = x.shape[0] if M is None else M
    N = x.shape[1] if N is None else N
    ld = x.stride(0) if ld is None else ld
    fn = lib().mdt_colsum_bf16 if x.dtype == bf16 else lib().mdt_colsum_f32
    check(fn(ptr(x), M, N, ld, ptr(out), stream_ptr()), "mdt_colsum")


def ln_modulate(x, shift, scale, ld_mod, rows_per_group, M, D, save_stats=True, eps=1e-6):
    out = torch.empty(M, D, dtype=bf16, device=x.device)
    mean = torch.empty(M, dtype=f32, device=x.device) if save_stats else None
    rstd = torch.empty(M, dtype=f32, device=x.device) if save_stats else None
    check(lib().mdt_ln_modulate(ptr(x), ptr(shift), ptr(scale), ld_mod, rows_per_group, ptr(out), ptr(mean),
                                ptr(rstd), M, D, eps, stream_ptr()), "mdt_ln_modulate")
    return out, mean, rstd


def ln_modulate_bwd(dxmod, x, mean, rstd, scale, ld_mod, rows_per_group, g, accumulate, dshift, dscale, ld_dmod, M, D):
    check(lib().mdt_ln_modulate_bwd(ptr(dxmod), ptr(x), ptr(mean), ptr(rstd), ptr(scale), ld_mod, rows_per_group,
                                    ptr(g), int(accumulate), ptr(dshift), ptr(dscale), ld_dmod, M, D, stream_ptr()),
          "mdt_ln_modulate_bwd")


def ln_modulate_bwd_gate(dxmod, x, mean, rstd, scale, ld_mod, rows_per_group, g, accumulate, dshift, dscale, ld_dmod,
                         M, D, gate_next=None):
    """LN-modulate backward; with `gate_next = (y, gate, ld_gate, dgate, ld_dgate, dbias)` also the gate backward of
    the branch that consumes the finished residual gradient (one pass over g).  Returns dy (bf16) or None."""
    dy = None
    y = gate = dgate = dbias = None
    ld_gate = ld_dgate = 0
    if gate_next is not None:
        y, gate, ld_gate, dgate, ld_dgate, dbias = gate_next
        dy = torch.empty(M, D, dtype=bf16, device=g.device)
    check(lib().mdt_ln_modulate_bwd_gate(ptr(dxmod), ptr(x), ptr(mean), ptr(rstd), ptr(scale), ld_mod, rows_per_group,
                                         ptr(g), int(accumulate), ptr(dshift), ptr(dscale), ld_dmod, ptr(y), ptr(gate),
                                         ld_gate, ptr(dy), ptr(dgate), ld_dgate, ptr(dbias), M, D, stream_ptr()),
          "mdt_ln_modulate_bwd_gate")
    return dy


def gate_bwd(g, y, gate, ld_gate, rows_per_group, dgate, ld_dgate, dbias, M, D):
    dy = torch.empty(M, D, dtype=bf16, device=g.device)
    check(lib().mdt_gate_bwd(ptr(g), ptr(y), ptr(gate), ld_gate, rows_per_group, ptr(dy), ptr(dgate), ld_dgate,
                             ptr(dbias), M, D, stream_ptr()), "mdt_gate_bwd")
    return dy


def attention_fwd(qkv, B, T, H, dh, need_lse=True):
    _c(qkv, bf16)
    out = torch.empty(B * T, H * dh, dtype=bf16, device=qkv.device)
    lse = torch.empty(2, B, H, T, dtype=f32, device=qkv.device) if need_lse else None  # [1] = scratch for delta
    check(lib().mdt_attention_fwd(ptr(qkv), ptr(out), ptr(lse), B, T, H, dh, stream_ptr()), "mdt_attention_fwd")
    return out, lse


def attention_bwd(qkv, out, dout, lse, B, T, H, dh):
    _c(qkv, bf16), _c(out, bf16), _c(dout, bf16), _c(lse, f32)
    dqkv = torch.empty_like(qkv)
    check(lib().mdt_attention_bwd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dqkv), B, T, H, dh, stream_ptr()),
          "mdt_attention_bwd", 2)
    return dqkv


def unmask_tokens(u, mask_token, pos, ids_restore, B, T, Lt, D):
    out = torch.empty(B, Lt, D, dtype=f32, device=u.device)
    check(lib().mdt_unmask_tokens(ptr(u), ptr(mask_token), ptr(pos), ptr(ids_restore), ptr(out), B, T, Lt, D,
                                  stream_ptr()), "mdt_unmask_tokens")
    return out


def unmask_tokens_bwd(g, ids_restore, dmask_token, B, T, Lt, D):
    du = torch.empty(B * T, D, dtype=bf16, device=g.device)
    check(lib().mdt_unmask_tokens_bwd(ptr(g), 0, ptr(ids_restore), ptr(du), ptr(dmask_token), B, T, Lt, D,
                                      stream_ptr()), "mdt_unmask_tokens_bwd")
    return du


def gather_rows_bf16(x, idx, B, T, Lt, D):
    """out[b*T + i] = x[b*Lt + idx[b, i]] for a bf16 x [B*Lt, D] and idx [B, T] int64 -> [B*T, D] bf16."""
    _c(x, bf16), _c(idx, torch.int64)
    out = torch.empty(B * T, D, dtype=bf16, device=x.device)
    check(lib().mdt_gather_rows_bf16(ptr(x), ptr(idx), ptr(out), B, T, Lt, D, stream_ptr()), "mdt_gather_rows_bf16")
    return out


def edm_loss(F, xin, y, sigma, mask, gl, sigma_data, mae_coef, p, want_D=False, want_dF=True):
    B, C, R, _ = xin.shape
    loss = torch.empty(B, dtype=f32, device=xin.device)
    Dx = torch.empty_like(xin) if want_D else None
    dF = torch.empty(F.shape, dtype=bf16, device=xin.device) if want_dF else None
    check(lib().mdt_edm_loss(ptr(F), ptr(xin), ptr(y), ptr(sigma), ptr(mask), ptr(gl), sigma_data, mae_coef,
                             ptr(loss), ptr(Dx), ptr(dF), B, C, R, p, stream_ptr()), "mdt_edm_loss")
    return loss, Dx, dF


def edm_loss_logvar(F, xin, y, sigma, mask, gl, sigma_data, mae_coef, p, freqs, phases, w, want_dF=True):
    """`edm_loss` with the learned weighting u(sigma) (mdt_edm_loss_logvar).  Returns (objective, loss, u, du, dF):
    objective = exp(-u) E + u + M, loss = E + M (`edm_loss`'s bits), u [B]; du [B] and dF only with `gl`."""
    B, C, R, _ = xin.shape
    dev = xin.device
    obj, loss, u = (torch.empty(B, dtype=f32, device=dev) for _ in range(3))
    du = torch.empty(B, dtype=f32, device=dev) if gl is not None else None
    dF = torch.empty(F.shape, dtype=bf16, device=dev) if want_dF else None
    check(lib().mdt_edm_loss_logvar(ptr(F), ptr(xin), ptr(y), ptr(sigma), ptr(mask), ptr(gl), sigma_data, mae_coef,
                                    ptr(freqs), ptr(phases), ptr(w), freqs.numel(), ptr(obj), ptr(loss), ptr(u),
                                    ptr(du), ptr(dF), B, C, R, p, stream_ptr()), "mdt_edm_loss_logvar")
    return obj, loss, u, du, dF


def logvar(sigma, freqs, phases, w):
    """u(sigma) [B] of the learned loss weighting (mdt_logvar)."""
    _c(sigma, f32), _c(freqs, f32), _c(phases, f32), _c(w, f32)
    u = torch.empty(sigma.numel(), dtype=f32, device=sigma.device)
    check(lib().mdt_logvar(ptr(sigma), ptr(freqs), ptr(phases), ptr(w), freqs.numel(), sigma.numel(), ptr(u),
                           stream_ptr()), "mdt_logvar")
    return u


def logvar_wgrad(sigma, freqs, phases, du, dw):
    """dw[j] += sum_b du[b] phi_j(c_b) in a fixed order (mdt_logvar_wgrad)."""
    _c(sigma, f32), _c(freqs, f32), _c(phases, f32), _c(du, f32), _c(dw, f32)
    check(lib().mdt_logvar_wgrad(ptr(sigma), ptr(freqs), ptr(phases), ptr(du), freqs.numel(), sigma.numel(), ptr(dw),
                                 stream_ptr()), "mdt_logvar_wgrad")


def step_front(moments, eps, rnd_normal, noise_unit, labels=None, drop_u=None, drop_prob=0.0, scale_factor=0.18215,
               P_mean=-1.2, P_std=1.2):
    """moments -> latent, label dropout (in place on `labels`), sigma draw, noise injection: one launch.
    Returns (y, yn, sigma)."""
    _c(moments, f32), _c(eps, f32), _c(rnd_normal, f32), _c(noise_unit, f32), _c(labels, f32), _c(drop_u, f32)
    B, C2, R, _ = moments.shape
    C = C2 // 2
    y = torch.empty(B, C, R, R, dtype=f32, device=moments.device)
    yn = torch.empty_like(y)
    sigma = torch.empty(B, dtype=f32, device=moments.device)
    nc = labels.shape[1] if labels is not None else 0
    check(lib().mdt_step_front(ptr(moments), ptr(eps), ptr(rnd_normal), ptr(noise_unit), ptr(drop_u), drop_prob,
                               scale_factor, P_mean, P_std, ptr(y), ptr(yn), ptr(sigma),
                               ptr(labels) if drop_u is not None else 0, B, C, R, nc, stream_ptr()), "mdt_step_front")
    return y, yn, sigma


def flow_step_front(moments, eps, rnd_normal, noise_unit, labels=None, drop_u=None, drop_prob=0.0,
                    scale_factor=0.18215, P_mean=0.0, P_std=1.0):
    """`step_front` for rectified flow: moments -> latent x, label dropout, t = sigmoid(P_mean + P_std rnd_normal),
    x_t = (1 - t) x + t noise_unit: one launch.  Returns (x, x_t, t)."""
    _c(moments, f32), _c(eps, f32), _c(rnd_normal, f32), _c(noise_unit, f32), _c(labels, f32), _c(drop_u, f32)
    B, C2, R, _ = moments.shape
    C = C2 // 2
    y = torch.empty(B, C, R, R, dtype=f32, device=moments.device)
    xt = torch.empty_like(y)
    t = torch.empty(B, dtype=f32, device=moments.device)
    nc = labels.shape[1] if labels is not None else 0
    check(lib().mdt_flow_step_front(ptr(moments), ptr(eps), ptr(rnd_normal), ptr(noise_unit), ptr(drop_u), drop_prob,
                                    scale_factor, P_mean, P_std, ptr(y), ptr(xt), ptr(t),
                                    ptr(labels) if drop_u is not None else 0, B, C, R, nc, stream_ptr()),
          "mdt_flow_step_front")
    return y, xt, t


def flow_loss(F, xt, y, eps, t, mask, gl, mae_coef, p, want_xhat=False, want_dF=True):
    """Rectified-flow loss of the velocity F (mdt_flow_loss).  Returns (loss [B], x_hat or None, dF bf16 or None)."""
    B, C, R, _ = xt.shape
    loss = torch.empty(B, dtype=f32, device=xt.device)
    xh = torch.empty_like(xt) if want_xhat else None
    dF = torch.empty(F.shape, dtype=bf16, device=xt.device) if want_dF else None
    check(lib().mdt_flow_loss(ptr(F), ptr(xt), ptr(y), ptr(eps), ptr(t), ptr(mask), ptr(gl), mae_coef, ptr(loss),
                              ptr(xh), ptr(dF), B, C, R, p, stream_ptr()), "mdt_flow_loss")
    return loss, xh, dF


def ect_step_front(moments, eps, rnd_normal, noise_unit, qs, labels=None, drop_u=None, drop_prob=0.0,
                   scale_factor=0.18215, P_mean=-1.1, P_std=2.0, k=8.0, b=1.0):
    """`step_front` for Easy Consistency Tuning: moments -> latent x, label dropout, t = exp(P_mean + P_std rnd_normal),
    r = t max(0, 1 - qs (1 + k sigmoid(-b t))), x_t = x + t noise_unit, x_r = x + r noise_unit: one launch.  `qs` is
    one fp32 word on the device holding q^-(s+1).  Returns (x, x_t, x_r, sigma of the target forward, t, r)."""
    _c(moments, f32), _c(eps, f32), _c(rnd_normal, f32), _c(noise_unit, f32), _c(qs, f32), _c(labels, f32), \
        _c(drop_u, f32)
    B, C2, R, _ = moments.shape
    C = C2 // 2
    y = torch.empty(B, C, R, R, dtype=f32, device=moments.device)
    xt, xr = torch.empty_like(y), torch.empty_like(y)
    sr, t, r = (torch.empty(B, dtype=f32, device=moments.device) for _ in range(3))
    nc = labels.shape[1] if labels is not None else 0
    check(lib().mdt_ect_step_front(ptr(moments), ptr(eps), ptr(rnd_normal), ptr(noise_unit), ptr(drop_u), drop_prob,
                                   scale_factor, P_mean, P_std, ptr(qs), float(k), float(b), ptr(y), ptr(xt), ptr(xr),
                                   ptr(sr), ptr(t), ptr(r), ptr(labels) if drop_u is not None else 0, B, C, R, nc,
                                   stream_ptr()), "mdt_ect_step_front")
    return y, xt, xr, sr, t, r


def ect_loss(Ft, Fr, xt, xr, y, t, r, mask, gl, sigma_data, c, mae_coef, p, want_D=False, want_dF=True):
    """Consistency loss of the student output Ft against the target output Fr (mdt_ect_loss).  Returns (loss [B],
    D_t or None, dF bf16 or None)."""
    B, C, R, _ = xt.shape
    loss = torch.empty(B, dtype=f32, device=xt.device)
    D = torch.empty_like(xt) if want_D else None
    dF = torch.empty(Ft.shape, dtype=bf16, device=xt.device) if want_dF else None
    check(lib().mdt_ect_loss(ptr(Ft), ptr(Fr), ptr(xt), ptr(xr), ptr(y), ptr(t), ptr(r), ptr(mask), ptr(gl),
                             float(sigma_data), float(c), float(mae_coef), ptr(loss), ptr(D), ptr(dF), B, C, R, p,
                             stream_ptr()), "mdt_ect_loss")
    return loss, D, dF


def mg_loss(F, Fu, xin, y, sigma, labels, mask, gl, sigma_data, mae_coef, w, lo, hi, p, want_D=False, want_dF=True):
    """Model-guidance loss of the student output F against the guided target built with the null-label output Fu
    (mdt_mg_loss).  Returns (loss [B], the plain EDM loss [B], D or None, dF bf16 or None)."""
    B, C, R, _ = xin.shape
    loss, edm = torch.empty(B, dtype=f32, device=xin.device), torch.empty(B, dtype=f32, device=xin.device)
    D = torch.empty_like(xin) if want_D else None
    dF = torch.empty(F.shape, dtype=bf16, device=xin.device) if want_dF else None
    check(lib().mdt_mg_loss(ptr(F), ptr(Fu), ptr(xin), ptr(y), ptr(sigma), ptr(labels), labels.shape[1], ptr(mask),
                            ptr(gl), float(sigma_data), float(mae_coef), float(w), float(lo), float(hi), ptr(loss),
                            ptr(edm), ptr(D), ptr(dF), B, C, R, p, stream_ptr()), "mdt_mg_loss")
    return loss, edm, D, dF


def flow_mg_loss(F, Fu, xt, y, eps, t, labels, mask, gl, mae_coef, w, lo, hi, p, want_xhat=False, want_dF=True):
    """`mg_loss` on velocities (mdt_flow_mg_loss).  Returns (loss [B], the plain flow loss [B], x_hat or None, dF bf16
    or None)."""
    B, C, R, _ = xt.shape
    loss, plain = torch.empty(B, dtype=f32, device=xt.device), torch.empty(B, dtype=f32, device=xt.device)
    xh = torch.empty_like(xt) if want_xhat else None
    dF = torch.empty(F.shape, dtype=bf16, device=xt.device) if want_dF else None
    check(lib().mdt_flow_mg_loss(ptr(F), ptr(Fu), ptr(xt), ptr(y), ptr(eps), ptr(t), ptr(labels), labels.shape[1],
                                 ptr(mask), ptr(gl), float(mae_coef), float(w), float(lo), float(hi), ptr(loss),
                                 ptr(plain), ptr(xh), ptr(dF), B, C, R, p, stream_ptr()), "mdt_flow_mg_loss")
    return loss, plain, xh, dF


def flow_cfg_out(F, B, C, R, p, cfg_scale=None):
    """The velocity [B, C, R, R]: unpatchify(F), or with `cfg_scale` the CFG combine Fu + s (Fc - Fu) of F's two
    halves (cond rows first)."""
    out = torch.empty(B, C, R, R, dtype=f32, device=F.device)
    use = cfg_scale is not None
    check(lib().mdt_flow_cfg_out(ptr(F), int(use), float(cfg_scale) if use else 0.0, ptr(out), B, C, R, p,
                                 stream_ptr()), "mdt_flow_cfg_out")
    return out


def edm_precond_out(F, xin, sigma, sigma_data, p):
    B, C, R, _ = xin.shape
    Dx = torch.empty_like(xin)
    check(lib().mdt_edm_precond_out(ptr(F), ptr(xin), ptr(sigma), sigma_data, ptr(Dx), B, C, R, p, stream_ptr()),
          "mdt_edm_precond_out")
    return Dx


def edm_precond_out_bwd(gD, sigma, sigma_data, p):
    B, C, R, _ = gD.shape
    Lt = (R // p) ** 2
    dF = torch.empty(B * Lt, p * p * C, dtype=bf16, device=gD.device)
    check(lib().mdt_edm_precond_out_bwd(ptr(gD), ptr(sigma), sigma_data, ptr(dF), B, C, R, p, stream_ptr()),
          "mdt_edm_precond_out_bwd")
    return dF


def cfg_precond_out(F, xin, sigma, sigma_data, cfg_scale, p):
    B, C, R, _ = xin.shape
    Dx = torch.empty_like(xin)
    check(lib().mdt_cfg_precond_out(ptr(F), ptr(xin), ptr(sigma), sigma_data, cfg_scale, ptr(Dx), B, C, R, p,
                                    stream_ptr()), "mdt_cfg_precond_out")
    return Dx


def guided_precond_out(F_main, p_main, F_guide, p_guide, xin, sigma, sigma_data, w):
    """D = c_skip x + c_out (Fg + w (Fm - Fg)); each F token-major in its own network's patch size."""
    B, C, R, _ = xin.shape
    Dx = torch.empty_like(xin)
    check(lib().mdt_guided_precond_out(ptr(F_main), p_main, ptr(F_guide), p_guide, ptr(xin), ptr(sigma), sigma_data,
                                       w, ptr(Dx), B, C, R, stream_ptr()), "mdt_guided_precond_out")
    return Dx


def heun_update(mode, x_hat, denoised, d_cur, x_next, x_next_f32, t_hat, t_next):
    check(lib().mdt_heun_update(mode, ptr(x_hat), ptr(denoised), ptr(d_cur), ptr(x_next), ptr(x_next_f32),
                                float(t_hat), float(t_next), x_hat.numel(), stream_ptr()), "mdt_heun_update")


def lincomb_f64(a, x, b=0.0, y=None, c=0.0, z=None, out=None, out_f32=None, f32_scale=1.0):
    """out = a*x + b*y + c*z (x, y fp64; z fp32), out_f32 = float(out * f32_scale).  Returns (out, out_f32)."""
    _c(x, torch.float64), _c(y, torch.float64), _c(z, f32), _c(out, torch.float64), _c(out_f32, f32)
    check(lib().mdt_lincomb_f64(float(a), ptr(x), float(b), ptr(y), float(c), ptr(z), ptr(out), ptr(out_f32),
                                float(f32_scale), x.numel(), stream_ptr()), "mdt_lincomb_f64")
    return out, out_f32


def dpm_update(F, x, d_out, a, b0, h1=None, b1=0.0, h2=None, b2=0.0, velocity=False, t=0.0, out_f32=None):
    """One DPM-Solver++ step in place: D = F, or x - t F when `velocity` (a flow network's v^); d_out = D;
    x = a x + b0 D + b1 h1 + b2 h2 (terms with a None operand omitted); out_f32 = float(x)."""
    _c(F, f32), _c(x, torch.float64), _c(d_out, torch.float64), _c(h1, torch.float64), _c(h2, torch.float64)
    _c(out_f32, f32)
    for o in (F, d_out, h1, h2, out_f32):
        if o is not None and o.numel() != x.numel():
            raise L.MdtError(f"dpm_update operands must match the state's {x.numel()} elements, got {o.numel()}")
    check(lib().mdt_dpm_update(ptr(F), 1 if velocity else 0, float(t), ptr(x), ptr(d_out), ptr(h1), ptr(h2), float(a),
                               float(b0), float(b1), float(b2), ptr(out_f32), x.numel(), stream_ptr()),
          "mdt_dpm_update")
    return x, out_f32


def to_uint8_nhwc(img):
    """[B,C,H,W] f32 in [-1,1] -> uint8 [B,H,W,C] (sample.py:287)."""
    _c(img, f32)
    B, C, H, W = img.shape
    out = torch.empty(B, H, W, C, dtype=torch.uint8, device=img.device)
    check(lib().mdt_to_uint8_nhwc(ptr(img), ptr(out), B, C, H, W, stream_ptr()), "mdt_to_uint8_nhwc")
    return out


def adamw_ema(w, g, m, v, ema, w16, n, lr, step, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0,
              ema_decay=0.9999, grad_scale=1.0, max_blocks=0, coef=None):
    """coef (one fp32 word on the device, or None): the gradient scale becomes grad_scale * coef (a clip
    coefficient from `grad_clip_coef`)."""
    if coef is not None:
        _c(coef, f32)
        fn = lib().mdt_adamw_ema_coef_g16 if g.dtype == bf16 else lib().mdt_adamw_ema_coef
        check(fn(ptr(w), ptr(g), ptr(m), ptr(v), ptr(ema), ptr(w16), n, lr, beta1, beta2, eps, weight_decay, step,
                 ema_decay, grad_scale, ptr(coef), max_blocks, stream_ptr()), "mdt_adamw_ema_coef")
        return
    fn = lib().mdt_adamw_ema_g16 if g.dtype == bf16 else lib().mdt_adamw_ema   # bf16: all-reduced bf16 gradients
    check(fn(ptr(w), ptr(g), ptr(m), ptr(v), ptr(ema), ptr(w16), n, lr, beta1, beta2, eps, weight_decay, step,
             ema_decay, grad_scale, max_blocks, stream_ptr()), "mdt_adamw_ema")


# -- non-finite gradient guard: `flag` is one fp32 word (0 = finite), `counts` int64 {applied steps, skipped steps} --
def nonfinite_check(g, flag):
    """flag = 1 if any element of the fp32 tensor g is inf or NaN; leaves it alone otherwise (calls accumulate)."""
    _c(g, f32), _c(flag, f32)
    check(lib().mdt_nonfinite_check(ptr(g), g.numel(), ptr(flag), stream_ptr()), "mdt_nonfinite_check")


def cast_bf16_check(x, flag, out=None):
    """`cast_bf16` (same bits) that also sets `flag` if a stored bf16 value is inf or NaN."""
    _c(x, f32), _c(flag, f32), _c(out, bf16)
    if out is None:
        out = torch.empty(x.shape, dtype=bf16, device=x.device)
    check(lib().mdt_cast_f32_bf16_check(ptr(x), ptr(out), x.numel(), ptr(flag), stream_ptr()),
          "mdt_cast_f32_bf16_check")
    return out


def adamw_ema_guarded(w, g, m, v, ema, w16, n, lr, flag, counts, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=0.0,
                      ema_decay=0.9999, grad_scale=1.0, max_blocks=0, coef=None):
    """`adamw_ema` at step counts[0] + 1 when flag == 0; only the EMA update when flag != 0.  coef: as `adamw_ema`'s."""
    _c(flag, f32), _c(counts, torch.int64)
    if coef is not None:
        _c(coef, f32)
        fn = lib().mdt_adamw_ema_guarded_coef_g16 if g.dtype == bf16 else lib().mdt_adamw_ema_guarded_coef
        check(fn(ptr(w), ptr(g), ptr(m), ptr(v), ptr(ema), ptr(w16), n, lr, beta1, beta2, eps, weight_decay,
                 ema_decay, grad_scale, ptr(coef), ptr(flag), ptr(counts), max_blocks, stream_ptr()),
              "mdt_adamw_ema_guarded_coef")
        return
    fn = lib().mdt_adamw_ema_guarded_g16 if g.dtype == bf16 else lib().mdt_adamw_ema_guarded
    check(fn(ptr(w), ptr(g), ptr(m), ptr(v), ptr(ema), ptr(w16), n, lr, beta1, beta2, eps, weight_decay, ema_decay,
             grad_scale, ptr(flag), ptr(counts), max_blocks, stream_ptr()), "mdt_adamw_ema_guarded")


def optim_guard_advance(flag, counts):
    """counts[1 if flag else 0] += 1: once per step, after its last guarded optimizer pass."""
    _c(flag, f32), _c(counts, torch.int64)
    check(lib().mdt_optim_guard_advance(ptr(flag), ptr(counts), stream_ptr()), "mdt_optim_guard_advance")


# -- gradient-norm clipping: sums of squares in fp64 slots, then the norm and the clip coefficient (fp32 words) ---------
def grad_sumsq_scratch(n, device):
    """The fp64 scratch `grad_sumsq` needs for up to n elements (it may be shared by calls on one stream)."""
    k = lib().mdt_grad_sumsq_scratch(int(n))
    if k < 1:
        raise L.MdtError(f"mdt_grad_sumsq_scratch({n}) failed (status {k})")
    return torch.empty(k, dtype=torch.float64, device=device)


def grad_sumsq(g, out, scratch, flag=None):
    """out[0] = sum of g**2 (fp32 or bf16 g, fp64 sum in an order that depends on g.numel() alone); with `flag`, the
    non-finite check of `nonfinite_check` from the same read."""
    _c(g), _c(out, torch.float64), _c(scratch, torch.float64), _c(flag, f32)
    if g.dtype not in (f32, bf16):
        raise L.MdtError(f"grad_sumsq: expected float32 or bfloat16, got {g.dtype}")
    if scratch.numel() < lib().mdt_grad_sumsq_scratch(g.numel()):
        raise L.MdtError(f"grad_sumsq: {scratch.numel()} scratch slots for {g.numel()} elements (grad_sumsq_scratch)")
    check(lib().mdt_grad_sumsq(ptr(g), g.numel(), int(g.dtype == bf16), ptr(scratch), ptr(out), ptr(flag),
                               stream_ptr()), "mdt_grad_sumsq", 2)


def grad_clip_coef(sumsq, grad_scale, max_norm, norm, coef, flag=None):
    """norm = grad_scale * sqrt(sum(sumsq)) (fp64, rounded once), coef = min(1, max_norm / (norm + 1e-6)) as
    clip_grad_norm_ computes it (max_norm = inf: coef = 1); with `flag` and a finite max_norm a non-finite norm sets it."""
    _c(sumsq, torch.float64), _c(norm, f32), _c(coef, f32), _c(flag, f32)
    check(lib().mdt_grad_clip_coef(ptr(sumsq), sumsq.numel(), float(grad_scale), float(max_norm), ptr(norm),
                                   ptr(coef), ptr(flag), stream_ptr()), "mdt_grad_clip_coef")


def power_ema(w, emas, coeffs):
    """Power-function EMA profiles: emas[j] += coeffs[j] * (w - emas[j]) for up to 4 fp32 tensors of w's size, from one
    read of w.  `coeffs` are host floats (1 - beta_j), rounded to fp32 at the call."""
    import ctypes
    _c(w, f32)
    k = len(emas)
    if k != len(coeffs):
        raise L.MdtError(f"{k} profiles but {len(coeffs)} coefficients")
    for e in emas:
        _c(e, f32)
        if e.numel() != w.numel() or e.device != w.device:
            raise L.MdtError("every profile must have w's size and device")
    check(lib().mdt_power_ema(ptr(w), (ctypes.c_void_p * max(k, 1))(*[e.data_ptr() for e in emas]),
                              (ctypes.c_float * max(k, 1))(*[float(c) for c in coeffs]), k, w.numel(), stream_ptr()),
          "mdt_power_ema")


def copy_segments_f32(src, dst, seg):
    """dst[d:d + c] = src[s:s + c] for every row {s, d, c} of the int64 device table `seg` [k, 3] (fp32 elements of the
    flat tensors src and dst; the rows must not overlap in dst)."""
    _c(src, f32), _c(dst, f32), _c(seg, torch.int64)
    check(lib().mdt_copy_segments_f32(ptr(src), ptr(dst), ptr(seg), seg.shape[0], stream_ptr()),
          "mdt_copy_segments_f32")
