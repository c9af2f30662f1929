"""``B200MultiviewUNet`` -- drop-in for the reference's ``pipeline.unet`` (seam B-2, SURVEY.md section 8b).

Mirrors ``UNetMultiviewConditionModel`` (reference src/diffusers/models/unets/unet_multiview_condition.py:501-509):
same ``forward(sample, timestep, skeletons, domains, num_frames, return_dict)`` signature, ``.config`` attributes
the pipeline reads (``enable_pose_encoder``, ``time_cond_proj_dim``; pipeline_diffuman4d.py:151,230,392), ``.dtype``,
``.device``, ``.to()``.  All arithmetic runs in libd4d.so through the C ABI; there is no torch fallback.
"""
from __future__ import annotations

import ctypes as C
from types import SimpleNamespace
from typing import Dict, List, Optional, Union

import torch

from ._lib import D4DConfig, check, lib
from .config import UNetConfig

_DOMAIN_IDS = {"spatial": 0, "temporal": 1}
_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


class UNetMultiviewConditionOutput(SimpleNamespace):
    """Same field as the reference's output dataclass (``.sample``)."""


def _c_config(cfg: UNetConfig) -> D4DConfig:
    c = D4DConfig()
    c.in_channels, c.out_channels = cfg.in_channels, cfg.out_channels
    for i in range(4):
        c.block_out_channels[i] = cfg.block_out_channels[i]
        c.num_heads[i] = cfg.attention_head_dim[i]
        c.has_attn2[i] = int(cfg.has_attn2(i))
    c.layers_per_block = cfg.layers_per_block
    c.use_linear_projection = int(cfg.use_linear_projection)
    c.norm_num_groups = cfg.norm_num_groups
    c.norm_eps = cfg.norm_eps
    c.flip_sin_to_cos = int(cfg.flip_sin_to_cos)
    c.freq_shift = float(cfg.freq_shift)
    c.num_3d_attn_blocks = cfg.num_3d_attn_blocks
    c.enable_tem_embeds = int(cfg.enable_tem_embeds)
    c.enable_pose_encoder = int(cfg.enable_pose_encoder)
    c.center_input_sample = int(cfg.center_input_sample)
    return c


class B200MultiviewUNet:
    """The UNet of the Diffuman4D denoise step on one H100.  One instance per device (the reference drives one
    pipeline per GPU from its own thread, src/samplers/sampling_runner.py:26-43)."""

    def __init__(self, config: UNetConfig, device: Union[int, str, torch.device] = 0):
        self.config = config
        dev = torch.device(device if not isinstance(device, int) else f"cuda:{device}")
        if dev.type != "cuda":
            raise ValueError("B200MultiviewUNet runs on CUDA devices only (no CPU path exists)")
        self._device = torch.device("cuda", dev.index or 0)
        self._dtype = torch.bfloat16
        self._h = C.c_void_p()
        cc = _c_config(config)
        check(lib().d4d_create(C.byref(cc), self._device.index, C.byref(self._h)), "d4d_create")
        self._finalized = False

    # ---- nn.Module-like surface the reference pipeline touches ------------------------------------
    @property
    def dtype(self):
        return self._dtype

    @property
    def device(self):
        return self._device

    def to(self, *args, **kwargs):
        """Accepted for interface compatibility (``DiffusionPipeline.to``); the model is pinned to its GPU."""
        for a in list(args) + list(kwargs.values()):
            if isinstance(a, (str, torch.device)) and torch.device(a).type == "cuda":
                idx = torch.device(a).index
                if idx is not None and idx != self._device.index:
                    raise ValueError(f"this UNet was created on {self._device}; create a new one for {a}")
            if isinstance(a, torch.dtype) and a not in (torch.bfloat16,):
                raise ValueError("the CUDA path computes in bfloat16 only (reference default, configs/model/diffuman4d.yaml:4)")
        return self

    def eval(self):
        return self

    def expected_keys(self) -> List[str]:
        n = lib().d4d_num_weights(self._h)
        return [lib().d4d_weight_key(self._h, i).decode() for i in range(n)]

    # ---- weights ------------------------------------------------------------------------------------
    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """Load a diffusers-layout state_dict (keys of ``unet/diffusion_pytorch_model.safetensors``)."""
        expected = set(self.expected_keys())
        unexpected = [k for k in state_dict if k not in expected]
        missing = [k for k in expected if k not in state_dict]
        if strict and (unexpected or missing):
            raise RuntimeError(f"Error(s) in loading state_dict: missing {missing[:5]}{'...' if len(missing) > 5 else ''}, "
                               f"unexpected {unexpected[:5]}{'...' if len(unexpected) > 5 else ''}")
        for k, t in state_dict.items():
            if k not in expected:
                continue
            t = t.detach().cpu().contiguous()
            if t.dtype not in _DTYPE_CODE:
                t = t.float()
            shape = (C.c_int64 * max(t.dim(), 1))(*(list(t.shape) or [1]))
            check(lib().d4d_load_weight(self._h, k.encode(), t.data_ptr(), shape, max(t.dim(), 1),
                                        _DTYPE_CODE[t.dtype]), f"d4d_load_weight({k})")
        check(lib().d4d_finalize_weights(self._h), "d4d_finalize_weights")
        self._finalized = True
        return self

    @classmethod
    def from_state_dict(cls, config: UNetConfig, state_dict, device=0) -> "B200MultiviewUNet":
        return cls(config, device).load_state_dict(state_dict)

    # ---- forward ------------------------------------------------------------------------------------
    def forward(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int],
                skeletons: Optional[torch.Tensor] = None, domains: List[str] = None, num_frames: int = 1,
                return_dict: bool = True):
        cfg = self.config
        if sample.dim() != 4:
            raise ValueError("sample must be [B, C, H, W]")
        B, Cin, H, W = sample.shape
        if Cin != cfg.in_channels:
            raise ValueError(f"sample has {Cin} channels, config.in_channels = {cfg.in_channels}")
        if domains is None:
            if cfg.enable_tem_embeds:
                raise ValueError("domains is required when enable_tem_embeds")
            domains = ["spatial"] * max(1, B // max(num_frames, 1))
        if len(domains) * num_frames != B:
            raise ValueError(f"num_frames: {num_frames} * len(domains): {len(domains)} != len(emb): {B}")
        try:
            dom = (C.c_int32 * len(domains))(*[_DOMAIN_IDS[d] for d in domains])
        except KeyError as e:
            raise ValueError(f"Invalid domain for temporal embedding: {e.args[0]}") from None
        if not torch.is_tensor(timestep):
            timestep = torch.tensor([timestep], dtype=torch.int64, device=self._device)
        timestep = timestep.to(device=self._device, dtype=torch.int64).reshape(-1)
        if timestep.numel() == 1:
            timestep = timestep.expand(B)
        timestep = timestep.contiguous()
        sample = sample.to(device=self._device, dtype=torch.bfloat16).contiguous()
        if cfg.enable_pose_encoder:
            if skeletons is None:
                raise ValueError("skeletons are required when enable_pose_encoder")
            skeletons = skeletons.to(device=self._device, dtype=torch.bfloat16).contiguous()
            if tuple(skeletons.shape) != (B, 3, 8 * H, 8 * W):
                raise ValueError(f"skeletons must be [B, 3, 8H, 8W], got {tuple(skeletons.shape)}")
        out = torch.empty(B, cfg.out_channels, H, W, device=self._device, dtype=torch.bfloat16)
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream().cuda_stream
            check(lib().d4d_unet_forward(self._h, sample.data_ptr(), timestep.data_ptr(),
                                         skeletons.data_ptr() if cfg.enable_pose_encoder else None, dom, len(domains),
                                         B, num_frames, H, W, out.data_ptr(), stream), "d4d_unet_forward")
        if not return_dict:
            return (out,)
        return UNetMultiviewConditionOutput(sample=out)

    __call__ = forward

    def debug_taps(self, sample, timestep, skeletons=None, domains=None, num_frames: int = 1) -> Dict[str, torch.Tensor]:
        """Intermediate activations for drift reports: {"conv_in", "down_blocks.i", "mid_block", "up_blocks.i"} -> NCHW bf16.
        One (prefix of a) forward is run per tap (``d4d_debug_tap``); same argument checks as ``forward``."""
        cfg = self.config
        B, _, H, W = sample.shape
        dom = (C.c_int32 * len(domains))(*[_DOMAIN_IDS[d] for d in domains])
        sample = sample.to(device=self._device, dtype=torch.bfloat16).contiguous()
        timestep = timestep.to(device=self._device, dtype=torch.int64).reshape(-1).contiguous()
        if cfg.enable_pose_encoder:
            skeletons = skeletons.to(device=self._device, dtype=torch.bfloat16).contiguous()
        sk_ptr = skeletons.data_ptr() if cfg.enable_pose_encoder else None
        out: Dict[str, torch.Tensor] = {}
        name, dims = C.create_string_buffer(64), (C.c_int32 * 3)()
        with torch.cuda.device(self._device):
            stream = torch.cuda.current_stream().cuda_stream
            tap = 0
            while lib().d4d_debug_tap(self._h, sample.data_ptr(), timestep.data_ptr(), sk_ptr, dom, len(domains), B,
                                      num_frames, H, W, tap, None, name, dims, stream) == 0:
                t = torch.empty(B, dims[0], dims[1], dims[2], device=self._device, dtype=torch.bfloat16)
                check(lib().d4d_debug_tap(self._h, sample.data_ptr(), timestep.data_ptr(), sk_ptr, dom, len(domains), B,
                                          num_frames, H, W, tap, t.data_ptr(), name, dims, stream), "d4d_debug_tap")
                out[name.value.decode()] = t
                tap += 1
        return out

    def forward_launches(self, n_domains: int, B: int, F: int, h: int, w: int) -> int:
        n = C.c_int(0)
        check(lib().d4d_forward_launches(self._h, n_domains, B, F, h, w, C.byref(n)))
        return n.value

    def workspace_bytes(self, n_domains: int, B: int, F: int, h: int, w: int) -> int:
        n = C.c_size_t(0)
        check(lib().d4d_workspace_bytes(self._h, n_domains, B, F, h, w, C.byref(n)))
        return n.value

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                lib().d4d_destroy(self._h)
                self._h = C.c_void_p()
        except Exception:  # noqa: BLE001 - interpreter shutdown
            pass
