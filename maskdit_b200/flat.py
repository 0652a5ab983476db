"""Flat parameter storage for the H100 engine.

All parameters of an `EDMPrecond` live in ONE contiguous fp32 device buffer (trainable first, frozen pos-embeds
last); the module's `nn.Parameter`s are views into it, so `state_dict()/load_state_dict()/deepcopy/.parameters()`
behave exactly as for the reference module (SURVEY.md §8b) while the engine gets:
  * one flat gradient buffer  -> a single NCCL all-reduce (train.py:178 DDP replaced, SURVEY.md §8e);
  * one fused AdamW+EMA pass over flat buffers (train.py:141, helper.py:47-58);
  * a bf16 shadow with identical offsets for the tensor-core GEMMs;
  * all 38 adaLN projection matrices contiguous, so the modulation of every block is ONE GEMM per step
    (the conditioning vector c is shared by all blocks: models/maskdit.py:505-506,547-548).
The layout is the C step driver's (csrc/driver.cu `build_layout`): the store reads it from the driver's model handle.
"""
from __future__ import annotations

import math

import torch

from ._lib import MdtError

ALIGN = 64  # elements (256 B fp32 / 128 B bf16): the driver starts every tensor on this boundary


def _round_up(n, a=ALIGN):
    return (n + a - 1) // a * a


class FlatStore:
    """Owns the flat buffers of one module.  `attach(named_params)` (re)builds them on the params' device."""

    def __init__(self, model, named_shapes):
        """`model`: the `CEngine` whose C model handle lays out the blob; `named_shapes`: the module's parameter
        shapes, whose names and element counts must be the handle's tensors."""
        layout = model.tensors()
        for k in sorted(set(layout) ^ set(named_shapes)):
            where = "the driver's layout" if k in layout else "the module"
            raise MdtError(f"parameter {k} is only in {where}")
        self.offsets = {}      # key -> (offset, numel, shape), in blob order
        for k, (o, n) in layout.items():
            shp = tuple(named_shapes[k])
            if math.prod(shp) != n:
                raise MdtError(f"parameter {k}: the module's shape {shp} does not hold the driver's {n} elements")
            self.offsets[k] = (o, n, shp)
        self.n_train = model.param_count(trainable_only=True)   # elements in the trainable region
        self.n_total = model.param_count(trainable_only=False)
        # the adaLN projections lead the blob: all weights as one [NA, hidden] matrix, then all biases
        w0 = next(v for k, v in self.offsets.items() if "adaLN_modulation" in k and k.endswith("weight"))
        b0 = next(v for k, v in self.offsets.items() if "adaLN_modulation" in k and k.endswith("bias"))
        self.ada_w_range = (w0[0], model.NA, w0[2][1])   # (offset, rows, hidden)
        self.ada_b_range = (b0[0], model.NA)
        self.device = None
        self.w32 = None
        self.w16 = None
        self.grad = None
        self._versions = None

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
