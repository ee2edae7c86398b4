"""Registry-level components with the reference's constructor / forward contracts, each running on the CUDA engine:

  BACKBONE_REGISTRY            D2ViT(cfg, input_shape)          /root/reference/projects/HIPIE/hipie/backbone/vit.py:378-467
  SEM_SEG_HEADS_REGISTRY       MaskDINOHead(cfg, input_shape)   hipie/models/maskdino/meta_arch/maskdino_head.py:21-82
                               MaskDINOEncoder(cfg, input_shape) hipie/models/maskdino/pixel_decoder/maskdino_encoder.py:190-434
  TRANSFORMER_DECODER_REGISTRY MaskDINODecoder(cfg, in_channels, mask_classification)
                                                                 hipie/models/maskdino/transformer_decoder/maskdino_decoder.py:36-529

They exist so that code which assembles HIPIE from detectron2 registries (build_backbone(cfg), build_maskdino(cfg)) finds the
same names; `HIPIE_IMG` itself drives the engine directly.  State_dict keys are the reference's, relative to the component
(e.g. `blocks.0.attn.qkv.weight` for D2ViT, `pixel_decoder.input_proj.0.0.weight` for MaskDINOHead).
"""
from collections import OrderedDict, namedtuple

import torch
import torch.nn as nn

from .. import ops
from . import params as P
from .engine import Engine

ShapeSpec = namedtuple("ShapeSpec", ["channels", "height", "width", "stride"], defaults=(None, None, None, None))

_VIT_DIMS = {"ViT-Base": (768, 12, 12), "ViT-Large": (1024, 24, 16), "ViT-huge": (1280, 32, 16)}


class _EngineComponent(nn.Module):
    """Holds the slice of the HIPIE parameter set that lives under `prefix` and an Engine over it."""

    prefix = ""

    def __init__(self, hp, device, state_dict=None, seed=0):
        super().__init__()
        self.hp = hp
        self.device_ = torch.device(device)
        if self.device_.type != "cuda":
            raise RuntimeError("hipie_b200 components run on a CUDA (sm_90a) device only; there is no CPU path")
        full = P.random_state_dict(hp, seed=seed)
        self._keys = [k for k in full if k.startswith(self.prefix)]
        self._sd = OrderedDict((k[len(self.prefix):], full[k]) for k in self._keys)
        self.engine = None
        self.load_state_dict(state_dict if state_dict is not None else self._sd)

    @property
    def device(self):
        return self.device_

    def state_dict(self, *a, **k):
        return OrderedDict(self._sd)

    def load_state_dict(self, sd, strict=True):
        known = set(k[len(self.prefix):] for k in self._keys)
        canon = {}
        for k, v in sd.items():
            c = P.canonical_name(self.prefix + k, self.hp)            # aliases of shared modules -> their canonical key
            canon.setdefault(c[len(self.prefix):] if c.startswith(self.prefix) else k, v)
        missing = [k for k in known if k not in canon]
        unexpected = [k for k in canon if k not in known]
        if strict and (missing or unexpected):
            raise RuntimeError(f"load_state_dict: missing {missing[:5]} ({len(missing)}), unexpected {unexpected[:5]} ({len(unexpected)})")
        for k in known:
            if k in canon:
                if tuple(canon[k].shape) != tuple(self._sd[k].shape):
                    raise RuntimeError(f"size mismatch for {k}: {tuple(canon[k].shape)} vs {tuple(self._sd[k].shape)}")
                self._sd[k] = canon[k].detach().float().cpu()
        self.engine = Engine({self.prefix + k: v for k, v in self._sd.items()}, self.hp, self.device_)
        return missing


def _hp_from_cfg(cfg):
    from .hipie_img import hp_from_cfg
    try:
        return hp_from_cfg(cfg)
    except NotImplementedError:
        raise
    except Exception:
        # a backbone-only cfg (no DDETRS node): only the ViT geometry is needed
        dims = _VIT_DIMS[cfg.MODEL.VIT.NAME]
        return dict(backbone="vit", vit=dict(embed_dim=dims[0], depth=dims[1], num_heads=dims[2], window_size=14,
                                             window_block_indexes=(0, 1, 3, 4, 6, 7, 9, 10), img_size=1024, patch_size=16, pretrain_img_size=224))


class D2ViT(_EngineComponent):
    """forward(x: (B, 3, H, W) normalised image) -> {"res3", "res4", "res5"} NCHW fp32; H, W multiples of 32."""

    prefix = "detr.detr.backbone.0.backbone."

    def __init__(self, cfg=None, input_shape=None, hp=None, device=None, state_dict=None):
        hp = hp if hp is not None else _hp_from_cfg(cfg)
        super().__init__(hp, device or (cfg.MODEL.DEVICE if cfg is not None else "cuda"), state_dict)
        e = hp["vit"]["embed_dim"]
        self._out_features = ["res3", "res4", "res5"]
        self._out_feature_channels = {"res3": e // 2, "res4": e, "res5": e}
        self._out_feature_strides = {"res3": 8, "res4": 16, "res5": 32}
        self.num_channels = [e // 2, e, e]
        self.strides = [8, 16, 32]

    @property
    def size_divisibility(self):
        return 32

    def output_shape(self):
        return {n: ShapeSpec(channels=self._out_feature_channels[n], stride=self._out_feature_strides[n]) for n in self._out_features}

    @torch.no_grad()
    def forward(self, x):
        feats = self.engine.vit(x.to(self.device_).float().contiguous(), normalized=True)
        return {k: v[0].permute(0, 3, 1, 2) for k, v in feats.items()}


class MaskDINOHead(_EngineComponent):
    """forward(features: {"res3","res4","res5"} NCHW) -> (outputs, None): outputs = {"pred_logits" (B, Q, 256) class embeddings,
    "pred_masks" (B, Q, H/4, W/4), "pred_boxes" (B, Q, 4)} -- the eval outputs of MaskDINOHead.layers (:77-82)."""

    prefix = "detr.mask_dino."

    def __init__(self, cfg=None, input_shape=None, hp=None, device=None, state_dict=None):
        hp = hp if hp is not None else _hp_from_cfg(cfg)
        super().__init__(hp, device or (cfg.MODEL.DEVICE if cfg is not None else "cuda"), state_dict)

    @torch.no_grad()
    def forward(self, features, mask=None, targets=None, lang_feat_pool=None):
        feats = {}
        for k in ("res3", "res4", "res5"):
            f = features[k].to(self.device_).float().permute(0, 2, 3, 1).contiguous()
            feats[k] = (f, ops.add_split(f)[1])
        md = self.engine.maskdino(feats, feats["res3"][0].shape[0])
        return {"pred_logits": md["pred_logits_emb"], "pred_masks": md["pred_masks"], "pred_boxes": md["pred_boxes"]}, None

    layers = forward


class MaskDINOEncoder(MaskDINOHead):
    """The pixel decoder alone: forward_features(features) -> (mask_features (B, 256, H/4, W/4), out[0], multi_scale list)."""

    @torch.no_grad()
    def forward_features(self, features, masks=None):
        feats = {}
        for k in ("res3", "res4", "res5"):
            f = features[k].to(self.device_).float().permute(0, 2, 3, 1).contiguous()
            feats[k] = (f, ops.add_split(f)[1])
        B = feats["res3"][0].shape[0]
        md = self.engine.maskdino(feats, B, pixel_decoder_only=True)
        return md["mask_features"], md["multi_scale"][0], md["multi_scale"]


class MaskDINODecoder(MaskDINOHead):
    """Registered for name compatibility; the decoder runs inside MaskDINOHead.forward (it consumes the encoder's bf16 planes
    directly, there is no separate launch sequence worth exposing)."""
