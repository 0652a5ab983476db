"""YAML config + CLI helpers for the train.py / generate.py twins.

The reference's config files (configs/{train,finetune,test}/*.yaml, schema in SURVEY.md §5) are accepted unchanged;
OmegaConf is replaced by PyYAML + attribute access.  Known quirks handled: `model.mask_ratio_fn: cos4` in
configs/finetune/imagenet256-latent-cos.yaml is an alias the reference's helper does not know (helper.py:14);
test YAMLs lack `model.self_cond` / `model.mask_ratio_fn`.
"""
from __future__ import annotations

import math
import re

import yaml


class Node(dict):
    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        return v

    def get_path(self, path, default=None):
        cur = self
        for part in path.split("."):
            if not isinstance(cur, dict) or part not in cur:
                return default
            cur = cur[part]
        return cur


def _wrap(x):
    if isinstance(x, dict):
        return Node({k: _wrap(v) for k, v in x.items()})
    if isinstance(x, list):
        return [_wrap(v) for v in x]
    if isinstance(x, str) and x == "None":
        return None
    return x


def load_config(path_or_text: str) -> Node:
    text = open(path_or_text).read() if "\n" not in path_or_text else path_or_text
    return _wrap(yaml.safe_load(text))


def mask_ratio_schedule(name="constant", ratio_scale=0.5, ratio_min=0.0):
    """get_mask_ratio_fn (train_utils/helper.py:9-27): progress in [0,1] -> mask ratio."""
    m = re.fullmatch(r"cos(?:ine)?(\d)", name or "constant")
    if m:
        k = int(m.group(1))
        return lambda x: (ratio_scale - ratio_min) * math.cos(math.pi * x / 2) ** k + ratio_min
    if name == "exp":
        return lambda x: (ratio_scale - ratio_min) * math.exp(-x * 7) + ratio_min
    if name == "linear":
        return lambda x: (ratio_scale - ratio_min) * x + ratio_min
    if name in ("constant", None):
        return lambda x: ratio_scale
    raise ValueError(f"Unknown mask ratio function: {name}")


def parse_int_list(s):
    """'1,2,5-10' -> [1,2,5,...,10]  (utils.py:140-151)."""
    if isinstance(s, list):
        return s
    out = []
    for part in s.split(","):
        m = re.fullmatch(r"(\d+)-(\d+)", part)
        out.extend(range(int(m.group(1)), int(m.group(2)) + 1) if m else [int(part)])
    return out


def parse_float_none(s):
    return None if s is None or str(s).lower() == "none" else float(s)


def build_net(cfg: Node, **extra):
    """Precond_models[config.model.precond](...) exactly as train.py:123-131 / generate.py:31-40 call it, plus
    `model.logvar_channels` (the learned loss weighting, not in the reference's configs: default 0, off)."""
    from .maskdit import Precond_models
    m = cfg.model
    return Precond_models[m.precond](img_resolution=m.in_size, img_channels=m.in_channels, num_classes=m.num_classes,
                                     model_type=m.model_type, use_decoder=m.use_decoder,
                                     mae_loss_coef=m.mae_loss_coef, pad_cls_token=m.pad_cls_token,
                                     logvar_channels=int(m.get("logvar_channels", 0) or 0), **extra)


ECT_KEYS = ("stage_steps", "q", "k", "b", "P_mean", "P_std")
MG_KEYS = ("scale", "interval")
OBJECTIVE_BLOCKS = ("ect", "mg")


def build_loss(cfg: Node):
    """The training loss of a config: `Losses[model.precond]()` as train.py:137 builds it, or, with
    `train.objective: ect`, Easy Consistency Tuning (`Losses['ect']`) of an EDM network with the `train.ect` block's
    `stage_steps` (required), `q`, `k`, `b`, `P_mean` and `P_std`, or, with `train.objective: mg`, model guidance
    (`Losses['mg']`) of a class-conditional EDM or flow network with the `train.mg` block's `scale` (required, >= 1,
    the CFG-equivalent scale) and `interval: [lo, hi]` (the noise levels, or flow times, that are guided; default
    all).  An absent `train.objective` is the precond's own objective.  Raises ValueError for a combination that cannot
    train."""
    from .loss import Losses
    m, tr = cfg.model, cfg.get("train") or Node()
    obj = tr.get("objective", None)
    given = [k for k in OBJECTIVE_BLOCKS if tr.get(k, None) is not None]
    for k in given:
        if obj != k:
            what = "consistency tuning" if k == "ect" else "model guidance"
            raise ValueError(f"train.{k} configures {what}: set train.objective: {k}")
    if obj in (None, m.precond):
        return Losses[m.precond]()
    if obj not in OBJECTIVE_BLOCKS:
        raise ValueError(f"unknown train.objective {obj!r} (the precond's own, 'ect' or 'mg')")
    if int(m.get("logvar_channels", 0) or 0):
        raise ValueError(f"train.objective: {obj} does not train a learned loss weighting: drop model.logvar_channels")
    if obj == "mg":
        return _build_mg(m, tr.get("mg", None))
    if m.precond != "edm":
        raise ValueError(f"train.objective: ect tunes an EDM network, not model.precond: {m.precond}")
    block = dict(tr.get("ect", None) or {})
    unknown = sorted(set(block) - set(ECT_KEYS))
    if unknown:
        raise ValueError(f"unknown train.ect keys {unknown} (known: {list(ECT_KEYS)})")
    if block.get("stage_steps") is None:
        raise ValueError("train.objective: ect needs train.ect.stage_steps (steps per tuning stage)")
    return Losses["ect"](**block)


def _build_mg(m, block):
    from .loss import Losses
    if m.precond not in ("edm", "flow"):
        raise ValueError(f"train.objective: mg trains an EDM or flow network, not model.precond: {m.precond}")
    if not int(m.get("num_classes", 0) or 0):
        raise ValueError("train.objective: mg guides a class-conditional network: model.num_classes is 0")
    if not float(m.get("class_dropout_prob", 0) or 0) > 0:
        raise ValueError("train.objective: mg needs model.class_dropout_prob > 0: the null-label output it guides "
                         "against is only trained on the dropped labels")
    block = dict(block or {})
    unknown = sorted(set(block) - set(MG_KEYS))
    if unknown:
        raise ValueError(f"unknown train.mg keys {unknown} (known: {list(MG_KEYS)})")
    if block.get("scale") is None:
        raise ValueError("train.objective: mg needs train.mg.scale (the CFG-equivalent scale, >= 1)")
    interval = block.get("interval")
    if interval is not None:
        if not isinstance(interval, (list, tuple)) or len(interval) != 2:
            raise ValueError(f"train.mg.interval must be [lo, hi], got {interval!r}")
        interval = (float(interval[0]), float(interval[1]))
    return Losses["mg"](scale=float(block["scale"]), interval=interval)
