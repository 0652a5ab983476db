"""Flat parameter storage for the H100 engine.

All parameters of an `EDMPrecond` live in ONE contiguous fp32 device buffer (trainable first, frozen pos-embeds
last); the module's `nn.Parameter`s are views into it, so `state_dict()/load_state_dict()/deepcopy/.parameters()`
behave exactly as for the reference module (SURVEY.md §8b) while the engine gets:
  * one flat gradient buffer  -> a single NCCL all-reduce (train.py:178 DDP replaced, SURVEY.md §8e);
  * one fused AdamW+EMA pass over flat buffers (train.py:141, helper.py:47-58);
  * a bf16 shadow with identical offsets for the tensor-core GEMMs;
  * all 38 adaLN projection matrices contiguous, so the modulation of every block is ONE GEMM per step
    (the conditioning vector c is shared by all blocks: models/maskdit.py:505-506,547-548).
"""
from __future__ import annotations

import torch

ALIGN = 64  # elements (256 B fp32 / 128 B bf16): keeps every tensor TMA- and float4-aligned


def _round_up(n, a=ALIGN):
    return (n + a - 1) // a * a


def layout_order(keys):
    """Trainable layout: adaLN weights (encoder blocks, decoder_layer, decoder blocks, final) contiguous, then
    the matching biases contiguous, then everything else in registration order; frozen tensors last."""
    def ada_rank(k):
        parts = k.split(".")
        if "blocks" == parts[1]:
            return (0, int(parts[2]))
        if parts[1] == "decoder_layer":
            return (1, 0)
        if parts[1] == "decoder_blocks":
            return (2, int(parts[2]))
        return (3, 0)  # final_layer

    ada_w = sorted([k for k in keys if "adaLN_modulation" in k and k.endswith("weight")], key=ada_rank)
    ada_b = sorted([k for k in keys if "adaLN_modulation" in k and k.endswith("bias")], key=ada_rank)
    frozen = [k for k in keys if k.endswith("pos_embed")]
    rest = [k for k in keys if k not in ada_w and k not in ada_b and k not in frozen]
    return ada_w, ada_b, rest, frozen


class FlatStore:
    """Owns the flat buffers of one module.  `attach(named_params)` (re)builds them on the params' device."""

    def __init__(self):
        self.device = None
        self.offsets = {}      # key -> (offset, numel, shape)
        self.n_train = 0       # elements in the trainable region (multiple of ALIGN)
        self.n_total = 0
        self.w32 = None
        self.w16 = None
        self.grad = None
        self.ada_w_range = None  # (offset, rows) of the concatenated adaLN weight [rows, hidden]
        self.ada_b_range = None
        self._versions = None
        self._ptr0 = None

    # -- layout ------------------------------------------------------------------------------------------------
    def plan(self, named_shapes):
        keys = list(named_shapes.keys())
        ada_w, ada_b, rest, frozen = layout_order(keys)
        off = 0
        self.offsets = {}
        for group in (ada_w, ada_b, rest):
            for k in group:
                n = 1
                for s in named_shapes[k]:
                    n *= s
                self.offsets[k] = (off, n, tuple(named_shapes[k]))
                off += _round_up(n)
        self.n_train = off
        for k in frozen:
            n = 1
            for s in named_shapes[k]:
                n *= s
            self.offsets[k] = (off, n, tuple(named_shapes[k]))
            off += _round_up(n)
        self.n_total = off
        if ada_w:
            o0 = self.offsets[ada_w[0]][0]
            rows, cur = 0, o0
            hidden = named_shapes[ada_w[0]][1]
            for k in ada_w:
                o, n, shp = self.offsets[k]
                assert o == cur and shp[1] == hidden, "adaLN weights must be contiguous"
                rows += shp[0]
                cur += n  # n is a multiple of ALIGN for every registry model (6*D*D etc.)
                assert n % ALIGN == 0
            self.ada_w_range = (o0, rows, hidden)
            b0 = self.offsets[ada_b[0]][0]
            cur = b0
            for k in ada_b:
                o, n, _ = self.offsets[k]
                assert o == cur and n % ALIGN == 0, "adaLN biases must be contiguous"
                cur += n
            self.ada_b_range = (b0, rows)

    # -- storage -----------------------------------------------------------------------------------------------
    def is_attached(self, params: dict) -> bool:
        if self.w32 is None:
            return False
        base = self.w32.data_ptr()
        for k, p in params.items():
            o, n, shp = self.offsets[k]
            if p.data_ptr() != base + 4 * o or p.device != self.w32.device or not p.is_contiguous():
                return False
        return True

    def attach(self, params: dict, device):
        """Copy every parameter into a fresh flat buffer on `device` and re-point `.data` at the views."""
        self.device = torch.device(device)
        w32 = torch.zeros(self.n_total, dtype=torch.float32, device=self.device)
        with torch.no_grad():
            for k, p in params.items():
                o, n, shp = self.offsets[k]
                w32[o:o + n].view(shp).copy_(p.data)
                p.data = w32[o:o + n].view(shp)
                p.grad = None
        self.w32 = w32
        self.w16 = torch.empty(self.n_total, dtype=torch.bfloat16, device=self.device)
        self.grad = None
        self._versions = None

    def view32(self, key):
        o, n, shp = self.offsets[key]
        return self.w32[o:o + n].view(shp)

    def view16(self, key):
        o, n, shp = self.offsets[key]
        return self.w16[o:o + n].view(shp)

    def gview(self, key):
        o, n, shp = self.offsets[key]
        return self.grad[o:o + n].view(shp)

    def ensure_grad(self):
        if self.grad is None:
            self.grad = torch.zeros(self.n_train, dtype=torch.float32, device=self.device)
        return self.grad

    def prefix_range(self, prefix):
        """(lo, hi) element range of the non-adaLN trainable tensors whose key starts with `prefix` — contiguous by
        construction (registration order), used to all-reduce / step a block's gradients as soon as they are final."""
        items = sorted(v[:2] for k, v in self.offsets.items()
                       if k.startswith(prefix) and "adaLN_modulation" not in k and not k.endswith("pos_embed"))
        lo, cur = items[0][0], items[0][0]
        for o, n in items:
            assert o == cur, "prefix range is not contiguous"
            cur = o + _round_up(n)
        return lo, cur

    # -- bf16 shadow -------------------------------------------------------------------------------------------
    def versions(self, params: dict):
        return sum(p._version for p in params.values())

    def shadow_stale(self, params: dict) -> bool:
        return self._versions != self.versions(params)

    def mark_shadow_fresh(self, params: dict):
        self._versions = self.versions(params)
