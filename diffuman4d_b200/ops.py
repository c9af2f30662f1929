"""Op-level Python wrappers over the C ABI (one hot-path kernel each).  torch is used only for device memory
and the current stream; all arithmetic happens in libd4d.so."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence

import torch

from ._lib import check, lib


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bf16c(t: torch.Tensor, name: str):
    if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous CUDA bfloat16 tensor")


def _stats_ws(stats: Optional[torch.Tensor], n_img: int, C: int):
    """Pointer of a GroupNorm statistics workspace: contiguous CUDA int64 holding at least [n_img][C][2] words, which the
    kernel ADDS into (pass it zeroed).  None passes NULL (no statistics)."""
    if stats is None:
        return None
    if stats.dtype != torch.int64 or not stats.is_cuda or not stats.is_contiguous():
        raise ValueError("stats must be a contiguous CUDA int64 tensor")
    if stats.numel() < n_img * C * 2:
        raise ValueError(f"stats needs at least {n_img} x {C} x 2 words")
    return stats.data_ptr()


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, a2: Optional[torch.Tensor] = None,
         rowvec: Optional[torch.Tensor] = None, rows_per_image: int = 0, residual: Optional[torch.Tensor] = None,
         geglu: bool = False, act: int = 0, out_scale: float = 1.0, block_n: int = 0, stats: Optional[torch.Tensor] = None,
         stats_rows: int = 0) -> torch.Tensor:
    """out = act((a | a2) @ w.T + bias + rowvec[row // rows_per_image]) * out_scale + residual   (bf16, fp32 accumulate).
    With ``geglu`` the rows of ``w``/``bias`` must already be tile-interleaved (see ``interleave_geglu``);
    ``block_n`` = 0 picks the tile width, otherwise it must be a multiple of 16 that divides N.
    ``stats``: zeroed int64 [M // stats_rows, N, 2] that receives the GroupNorm statistics of ``out`` (image = row //
    stats_rows; stats_rows a multiple of 32 that divides M)."""
    _bf16c(a, "a"), _bf16c(w, "w")
    M, K1 = a.shape
    K2 = 0 if a2 is None else a2.shape[1]
    N = w.shape[0]
    if w.shape[1] != K1 + K2:
        raise ValueError("w must be [N, K1+K2]")
    out = torch.empty(M, N // 2 if geglu else N, device=a.device, dtype=torch.bfloat16)
    if bias is not None and bias.dtype != torch.float32:
        raise ValueError("bias must be float32")
    check(lib().d4d_op_gemm(_p(a), a.stride(0), K1, _p(a2), 0 if a2 is None else a2.stride(0), K2, _p(w), M, N,
                            _p(bias), _p(rowvec), 0 if rowvec is None else rowvec.stride(0), rows_per_image,
                            _p(residual), 0 if residual is None else residual.stride(0), _p(out), out.stride(0),
                            int(geglu), act, float(out_scale), block_n,
                            _stats_ws(stats, M // stats_rows if stats_rows > 0 else 0, N), stats_rows, _stream()),
          "d4d_op_gemm")
    return out


def gemm_kv_scatter(a: torch.Tensor, w: torch.Tensor, *, kv_col0: int, rows_local: int, rows_global: int, row_offset: int,
                    dst: List[torch.Tensor], out: Optional[torch.Tensor] = None, block_n: int = 0) -> torch.Tensor:
    """QKV projection of a frame-sharded 3-D attention layer: ``a @ w.T`` with its columns >= ``kv_col0`` (K|V) stored
    into every buffer of ``dst`` (one per rank, 1 to 8) instead of ``out``.  Local row m of CFG half h = m // rows_local
    lands at row h * rows_global + row_offset + m % rows_local of each [halves * rows_global, ld] buffer.  Returns ``out``
    [M, N], whose columns < kv_col0 hold Q; its K|V columns are left as they were."""
    _bf16c(a, "a"), _bf16c(w, "w")
    M, K = a.shape
    N = w.shape[0]
    if w.shape[1] != K:
        raise ValueError("w must be [N, K]")
    if not 1 <= len(dst) <= 8:
        raise ValueError("dst must hold 1 to 8 buffers (one per rank)")
    ld = dst[0].stride(0)
    for t in dst:
        if t.dtype != torch.bfloat16 or not t.is_cuda or t.dim() != 2 or t.stride(1) != 1 or t.stride(0) != ld:
            raise ValueError("dst buffers must be row-major CUDA bfloat16 [rows, ld] matrices with one leading dimension")
        if t.shape[1] < N - kv_col0 or (rows_local > 0 and t.shape[0] < -(-M // rows_local) * rows_global):
            raise ValueError(f"dst buffers need [{-(-M // max(rows_local, 1))} * {rows_global}, {N - kv_col0}] elements")
    if out is None:
        out = torch.empty(M, N, device=a.device, dtype=torch.bfloat16)
    elif out.dtype != torch.bfloat16 or not out.is_cuda or out.shape != (M, N) or out.stride(1) != 1:
        raise ValueError(f"out must be a row-major CUDA bfloat16 [{M}, {N}] matrix")
    ptrs = (C.c_void_p * len(dst))(*[t.data_ptr() for t in dst])
    check(lib().d4d_op_gemm_kv_scatter(_p(a), a.stride(0), K, _p(w), M, N, _p(out), out.stride(0), kv_col0, ld, rows_local,
                                       rows_global, row_offset, len(dst), ptrs, block_n, _stream()),
          "d4d_op_gemm_kv_scatter")
    return out


def interleave_geglu(w: torch.Tensor, bias: torch.Tensor):
    """Re-order the rows of a GEGLU projection [2*inner, C] (a rows then g rows) in groups of 8: rows 16p..16p+7 are
    a[8p:8p+8], rows 16p+8..16p+15 the matching g rows (same transform the C++ weight loader applies).  The layout does
    not depend on the GEMM tile width.  Returns the re-ordered weight and bias."""
    N = w.shape[0]
    inner = N // 2
    idx = []
    for p in range(inner // 8):
        idx += list(range(8 * p, 8 * p + 8)) + list(range(inner + 8 * p, inner + 8 * p + 8))
    idx = torch.tensor(idx, device=w.device)
    return w[idx].contiguous(), bias[idx].contiguous()


def conv3x3(x_nhwc: torch.Tensor, w_octi: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
            rowvec: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None, act: int = 0,
            block_n: int = 0, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 conv on NHWC activations.  ``w_octi``: [Cout, 9, Cin] (tap = ky*3+kx).
    ``stats``: zeroed int64 [n, Cout, 2] that receives the GroupNorm statistics of the output."""
    _bf16c(x_nhwc, "x"), _bf16c(w_octi, "w")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_octi.shape[0]
    out = torch.empty(n, H, W, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    check(lib().d4d_op_conv3x3(_p(x_nhwc), n, H, W, Cin, _p(w_octi), Cout, _p(bias), _p(rowvec),
                               0 if rowvec is None else rowvec.stride(0), _p(residual), act, _p(out), block_n,
                               _stats_ws(stats, n, Cout), _stream()), "d4d_op_conv3x3")
    return out


def conv_weight_to_octi(w_oihw: torch.Tensor) -> torch.Tensor:
    co, ci, kh, kw = w_oihw.shape
    return w_oihw.permute(0, 2, 3, 1).reshape(co, kh * kw, ci).contiguous()


def attention(qkv: torch.Tensor, batch: int, seq: int, heads: int, head_dim: int, scale: float, *,
              kv: Optional[torch.Tensor] = None) -> torch.Tensor:
    """qkv: [batch*seq, 3*heads*head_dim] (q | k | v column blocks, head-major inside each).  Returns [batch*seq, heads*head_dim].
    ``kv``: keys and values from a separate [batch*seq_kv, 2*heads*head_dim] matrix (k | v column blocks; batch entry b
    owns rows [b*seq_kv, (b+1)*seq_kv)), as the frame-sharded window gathers them; qkv then supplies only the queries."""
    _bf16c(qkv, "qkv")
    C = heads * head_dim
    if qkv.shape != (batch * seq, 3 * C):
        raise ValueError("qkv shape")
    out = torch.empty(batch * seq, C, device=qkv.device, dtype=torch.bfloat16)
    base = qkv.data_ptr()
    k, v, seq_kv, ld_kv = base + 2 * C, base + 4 * C, 0, 0
    if kv is not None:
        _bf16c(kv, "kv")
        if kv.dim() != 2 or kv.shape[1] != 2 * C or kv.shape[0] % batch != 0 or kv.shape[0] == 0:
            raise ValueError("kv must be [batch*seq_kv, 2*heads*head_dim]")
        k, v, seq_kv, ld_kv = kv.data_ptr(), kv.data_ptr() + 2 * C, kv.shape[0] // batch, kv.stride(0)
    check(lib().d4d_op_attention(base, k, v, qkv.stride(0), _p(out), C, batch, seq, heads, head_dim, float(scale),
                                 seq_kv, ld_kv, _stream()), "d4d_op_attention")
    return out


def groupnorm(x1: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool,
              x2: Optional[torch.Tensor] = None, *, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x1: [n_img, hw, C1] (+ x2 [n_img, hw, C2] virtually concatenated on channels) -> [n_img, hw, C1+C2].
    ``stats``: zeroed int64 [n_img, C1+C2, 2] that keeps the statistics the norm computed (allocated when None)."""
    _bf16c(x1, "x1")
    n_img, hw, C1 = x1.shape
    C2 = 0 if x2 is None else x2.shape[2]
    out = torch.empty(n_img, hw, C1 + C2, device=x1.device, dtype=torch.bfloat16)
    if stats is None:
        stats = torch.zeros(n_img, C1 + C2, 2, device=x1.device, dtype=torch.int64)
    check(lib().d4d_op_groupnorm(_p(x1), C1, _p(x2), C2, n_img, hw, groups, float(eps), _p(gamma), _p(beta),
                                 int(silu), _p(out), _stats_ws(stats, n_img, C1 + C2), _stream()), "d4d_op_groupnorm")
    return out


def conv3x3_stride2(x_nhwc: torch.Tensor, w_octi: torch.Tensor, bias: Optional[torch.Tensor] = None, *,
                    stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3 / stride 2 / pad 1 conv (Downsample2D) through a strided tensor map: [n,H,W,Cin] -> [n,H/2,W/2,Cout].
    ``stats``: zeroed int64 [n, Cout, 2] that receives the GroupNorm statistics of the output."""
    _bf16c(x_nhwc, "x"), _bf16c(w_octi, "w")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_octi.shape[0]
    out = torch.empty(n, H // 2, W // 2, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    check(lib().d4d_op_conv_resample(_p(x_nhwc), n, H, W, Cin, _p(w_octi), Cout, _p(bias), 1, 0, 0, _p(out),
                                     _stats_ws(stats, n, Cout), _stream()), "d4d_op_conv_resample")
    return out


def upsample_phase_weights(w_oihw: torch.Tensor):
    """The four sub-pixel phase kernels [Cout, 4, Cin] (tap = ty*2+tx) of `nearest x2 -> conv3x3(w)`: output pixel
    (2y+a, 2x+b) sees rows {-1, 0} with weights {w0, w1+w2} for a = 0 and rows {0, +1} with {w0+w1, w2} for a = 1 (columns
    alike).  Same transform the C++ weight loader applies (csrc/unet.cu)."""
    w = w_oihw.float()
    rows = [[w[:, :, 0], w[:, :, 1] + w[:, :, 2]], [w[:, :, 0] + w[:, :, 1], w[:, :, 2]]]   # [a][ty] -> [Cout, Cin, 3(kx)]
    out = []
    for a in range(2):
        for b in range(2):
            taps = []
            for ty in range(2):
                r = rows[a][ty]
                cols = [r[:, :, 0], r[:, :, 1] + r[:, :, 2]] if b == 0 else [r[:, :, 0] + r[:, :, 1], r[:, :, 2]]
                taps += cols
            out.append(torch.stack(taps, dim=1).to(torch.bfloat16).contiguous())      # [Cout, 4, Cin]
    return out


def upsample2x_conv3x3(x_nhwc: torch.Tensor, w_oihw: torch.Tensor, bias: Optional[torch.Tensor] = None,
                       single_launch: bool = True, *, stats: Optional[torch.Tensor] = None) -> torch.Tensor:
    """nearest x2 upsample followed by a 3x3 / pad 1 conv (Upsample2D) as four sub-pixel phases on the low-res input.
    ``stats``: zeroed int64 [n, Cout, 2] that receives the GroupNorm statistics of the output."""
    _bf16c(x_nhwc, "x")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_oihw.shape[0]
    out = torch.empty(n, 2 * H, 2 * W, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    phases = upsample_phase_weights(w_oihw)
    st = _stats_ws(stats, n, Cout)
    if single_launch:
        wp = torch.stack(phases).contiguous()                                          # [4, Cout, 4, Cin]
        check(lib().d4d_op_conv_resample(_p(x_nhwc), n, H, W, Cin, _p(wp), Cout, _p(bias), 3, 0, 0, _p(out), st,
                                         _stream()), "d4d_op_conv_resample")
        return out
    for ph, wp in enumerate(phases):
        check(lib().d4d_op_conv_resample(_p(x_nhwc), n, H, W, Cin, _p(wp), Cout, _p(bias), 2, ph >> 1, ph & 1, _p(out),
                                         st, _stream()), "d4d_op_conv_resample")
    return out


def conv3x3_groupnorm(x_nhwc: torch.Tensor, w_octi: torch.Tensor, bias: Optional[torch.Tensor], gamma: torch.Tensor,
                      beta: torch.Tensor, groups: int, eps: float, silu: bool, residual: Optional[torch.Tensor] = None, *,
                      stats: Optional[torch.Tensor] = None):
    """conv3x3 whose epilogue accumulates the GroupNorm statistics of its output + the GroupNorm(+SiLU) that consumes them
    (no statistics pass).  Returns (conv_out, gn_out), both [n, H, W, Cout].  ``stats``: zeroed int64 [n, Cout, 2] that
    keeps the statistics (allocated when None)."""
    _bf16c(x_nhwc, "x"), _bf16c(w_octi, "w")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_octi.shape[0]
    conv_out = torch.empty(n, H, W, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    gn_out = torch.empty_like(conv_out)
    if stats is None:
        stats = torch.zeros(n, Cout, 2, device=x_nhwc.device, dtype=torch.int64)
    check(lib().d4d_op_conv3x3_groupnorm(_p(x_nhwc), n, H, W, Cin, _p(w_octi), Cout, _p(bias), _p(residual), groups,
                                         float(eps), _p(gamma), _p(beta), int(silu), _p(conv_out), _p(gn_out),
                                         _stats_ws(stats, n, Cout), _stream()), "d4d_op_conv3x3_groupnorm")
    return conv_out, gn_out


def pose_conv_weights(w_oihw: torch.Tensor) -> torch.Tensor:
    """The pose-encoder conv weight layouts of ``pose_conv0`` / ``pose_conv`` (same transform the C++ weight loader
    applies, csrc/unet.cu).  conv_layers.0 ([3, 3, 3, 3]) -> [9, 3, 3] = [tap][Cin][Cout]; conv_layers.2/4/6/8 ->
    [Cout, k*k*cp + 8] with column tap*cp + ci (tap = ky*k+kx), cp = max(Cin, 4): 4 for conv_layers.2 (Cin 3, zero
    weights for the pad channel), Cin for the others; and 8 zero columns that skew the rows over the shared-memory banks."""
    co, ci, k, _ = w_oihw.shape
    w = w_oihw.float()
    if (co, ci, k) == (3, 3, 3):
        return w.permute(2, 3, 1, 0).reshape(9, 3, 3).to(torch.bfloat16).contiguous()
    cp = max(ci, 4)
    out = torch.zeros(co, k * k, cp, device=w.device)
    out[:, :, :ci] = w.permute(0, 2, 3, 1).reshape(co, k * k, ci)
    out = torch.cat([out.reshape(co, k * k * cp), torch.zeros(co, 8, device=w.device)], 1)
    return out.to(torch.bfloat16).contiguous()


def pose_conv0(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor) -> torch.Tensor:
    """Pose encoder conv_layers.0 + SiLU: NCHW skeletons x [n, 3, H, W] -> NHWC [n, H, W, 4] with channel 3 = 0.
    ``w_packed`` from ``pose_conv_weights``; ``bias`` fp32 [3]."""
    _bf16c(x, "x"), _bf16c(w_packed, "w")
    if x.dim() != 4 or x.shape[1] != 3 or w_packed.numel() != 81:
        raise ValueError("pose_conv0 needs x [n, 3, H, W] and packed weights [9, 3, 3]")
    if bias.dtype != torch.float32 or bias.numel() != 3:
        raise ValueError("bias must be float32 [3]")
    n, _, H, W = x.shape
    out = torch.empty(n, H, W, 4, device=x.device, dtype=torch.bfloat16)
    check(lib().d4d_op_pose_conv0(_p(x), n, H, W, _p(w_packed), _p(bias), _p(out), _stream()), "d4d_op_pose_conv0")
    return out


def pose_conv(x: torch.Tensor, w_packed: torch.Tensor, bias: torch.Tensor, ksize: int, stride: int) -> torch.Tensor:
    """Pose encoder conv_layers.2/4/6/8 + SiLU (pad 1) on NHWC x [n, H, W, Cin] -> [n, Ho, Wo, Cout].  Cin is 4 for
    conv_layers.2, which reads conv_layers.0's padded pixels.  ``w_packed`` [Cout, k*k*Cin + 8] from
    ``pose_conv_weights``; ``bias`` fp32 [Cout]."""
    _bf16c(x, "x"), _bf16c(w_packed, "w")
    n, H, W, Cin = x.shape
    Cout = w_packed.shape[0]
    if w_packed.dim() != 2 or w_packed.shape[1] != ksize * ksize * Cin + 8:
        raise ValueError("w must be [Cout, ksize*ksize*Cin + 8]")
    if bias.dtype != torch.float32 or bias.numel() != Cout:
        raise ValueError("bias must be float32 [Cout]")
    Ho, Wo = (H + 2 - ksize) // stride + 1, (W + 2 - ksize) // stride + 1
    out = torch.empty(n, Ho, Wo, Cout, device=x.device, dtype=torch.bfloat16)
    check(lib().d4d_op_pose_conv(_p(x), n, Cin, H, W, _p(w_packed), _p(bias), Cout, ksize, stride, _p(out), _stream()),
          "d4d_op_pose_conv")
    return out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    _bf16c(x, "x")
    rows, C = x.shape
    out = torch.empty_like(x)
    check(lib().d4d_op_layernorm(_p(x), rows, C, float(eps), _p(gamma), _p(beta), _p(out), _stream()),
          "d4d_op_layernorm")
    return out


def _multistep_step(entry: str, noise, latents, cond_mask, timestep_indices, planes, lower_order_nums, sched,
                    guidance_scale, cfg):
    """``cfg_dpm_step`` / ``cfg_unipc_step`` / ``cfg_pndm_step`` / ``cfg_deis_step`` / ``cfg_dpm_single_step``:
    ``planes`` are the (name, bf16 [F,4,h,w] tensor or None) state planes in the order ``entry`` takes them."""
    _bf16c(noise, "noise"), _bf16c(latents, "latents"), _bf16c(cond_mask, "cond_mask")
    F, _, h, w = latents.shape
    for name, t in planes:
        if t is not None:
            _bf16c(t, name)
            if t.shape != latents.shape:
                raise ValueError(f"{name} must have the shape of latents")
    if lower_order_nums.dtype != torch.int32 or not lower_order_nums.is_cuda or lower_order_nums.numel() != F:
        raise ValueError("lower_order_nums must be a CUDA int32 [F] tensor")
    if timestep_indices.dtype != torch.int64 or not timestep_indices.is_cuda or timestep_indices.numel() != F:
        raise ValueError("timestep_indices must be a CUDA int64 [F] tensor")
    out = torch.empty_like(latents)
    ti_out = torch.empty_like(timestep_indices)
    lon_out = torch.empty_like(lower_order_nums)
    check(getattr(lib(), entry)(_p(noise), _p(latents), _p(cond_mask), _p(timestep_indices), _p(ti_out),
                                *(_p(t) for _, t in planes), _p(lower_order_nums), _p(lon_out), C.byref(sched),
                                float(guidance_scale), int(cfg), F, h, w, _p(out), _stream()), entry)
    return out, ti_out, lon_out


def cfg_dpm_step(noise: torch.Tensor, latents: torch.Tensor, cond_mask: torch.Tensor, timestep_indices: torch.Tensor,
                 x0_prev: torch.Tensor, lower_order_nums: torch.Tensor, sched, guidance_scale: float, cfg: bool):
    """One CFG + DPM-Solver++ step of F frames (``sched``: a ``d4d_dpm_sched`` from ``DPMSolverTables.c_struct``).
    ``noise`` [(cfg?2:1)*F,4,h,w]; ``x0_prev`` [F,4,h,w] bf16 is updated in place.  Returns (new latents, advanced
    timestep indices, advanced ``lower_order_nums``)."""
    return _multistep_step("d4d_cfg_dpm_step", noise, latents, cond_mask, timestep_indices, [("x0_prev", x0_prev)],
                           lower_order_nums, sched, guidance_scale, cfg)


def cfg_unipc_step(noise: torch.Tensor, latents: torch.Tensor, cond_mask: torch.Tensor, timestep_indices: torch.Tensor,
                   x0_prev: torch.Tensor, x0_prev2: Optional[torch.Tensor], last_sample: torch.Tensor,
                   lower_order_nums: torch.Tensor, sched, guidance_scale: float, cfg: bool):
    """One CFG + UniPC step of F frames (``sched``: a ``d4d_unipc_sched`` from ``UniPCTables.c_struct``).  ``noise``
    [(cfg?2:1)*F,4,h,w]; ``x0_prev``, ``x0_prev2`` (None at solver_order 1) and ``last_sample`` [F,4,h,w] bf16 are updated
    in place.  Returns (new latents, advanced timestep indices, advanced ``lower_order_nums``)."""
    return _multistep_step("d4d_cfg_unipc_step", noise, latents, cond_mask, timestep_indices,
                           [("x0_prev", x0_prev), ("x0_prev2", x0_prev2), ("last_sample", last_sample)], lower_order_nums,
                           sched, guidance_scale, cfg)


def cfg_pndm_step(noise: torch.Tensor, latents: torch.Tensor, cond_mask: torch.Tensor, timestep_indices: torch.Tensor,
                  ets: Sequence[torch.Tensor], cur_sample: torch.Tensor, counter: torch.Tensor, sched,
                  guidance_scale: float, cfg: bool):
    """One CFG + PNDM step of F frames (``sched``: a ``d4d_pndm_sched`` from ``PNDMTables.c_struct``).  ``noise``
    [(cfg?2:1)*F,4,h,w]; the four ``ets`` planes and ``cur_sample`` [F,4,h,w] bf16 are updated in place.  Returns (new
    latents, advanced timestep indices, advanced ``counter``)."""
    if len(ets) != 4:
        raise ValueError("ets must be the four planes ets0 .. ets3")
    return _multistep_step("d4d_cfg_pndm_step", noise, latents, cond_mask, timestep_indices,
                           [*((f"ets{i}", t) for i, t in enumerate(ets)), ("cur_sample", cur_sample)], counter, sched,
                           guidance_scale, cfg)


def cfg_deis_step(noise: torch.Tensor, latents: torch.Tensor, cond_mask: torch.Tensor, timestep_indices: torch.Tensor,
                  m_prev: torch.Tensor, m_prev2: Optional[torch.Tensor], lower_order_nums: torch.Tensor, sched,
                  guidance_scale: float, cfg: bool):
    """One CFG + DEIS step of F frames (``sched``: a ``d4d_deis_sched`` from ``DEISTables.c_struct``).  ``noise``
    [(cfg?2:1)*F,4,h,w]; ``m_prev`` and ``m_prev2`` (None below solver_order 3) [F,4,h,w] bf16 are updated in place.
    Returns (new latents, advanced timestep indices, advanced ``lower_order_nums``)."""
    return _multistep_step("d4d_cfg_deis_step", noise, latents, cond_mask, timestep_indices,
                           [("m_prev", m_prev), ("m_prev2", m_prev2)], lower_order_nums, sched, guidance_scale, cfg)


def cfg_dpm_single_step(noise: torch.Tensor, latents: torch.Tensor, cond_mask: torch.Tensor,
                        timestep_indices: torch.Tensor, x0_prev: torch.Tensor, x0_prev2: Optional[torch.Tensor],
                        cur_sample: torch.Tensor, lower_order_nums: torch.Tensor, sched, guidance_scale: float, cfg: bool):
    """One CFG + DPM-Solver++ singlestep step of F frames (``sched``: a ``d4d_dpm_single_sched`` from
    ``DPMSingleTables.c_struct``).  ``noise`` [(cfg?2:1)*F,4,h,w]; ``x0_prev``, ``x0_prev2`` (None below solver_order 3)
    and ``cur_sample`` [F,4,h,w] bf16 are updated in place.  Returns (new latents, advanced timestep indices, advanced
    ``lower_order_nums``)."""
    return _multistep_step("d4d_cfg_dpm_single_step", noise, latents, cond_mask, timestep_indices,
                           [("x0_prev", x0_prev), ("x0_prev2", x0_prev2), ("cur_sample", cur_sample)], lower_order_nums,
                           sched, guidance_scale, cfg)


def cfg_ddpm_step(noise: torch.Tensor, latents: torch.Tensor, cond_mask: torch.Tensor, timestep_indices: torch.Tensor,
                  frame_ids: torch.Tensor, sched, guidance_scale: float, cfg: bool):
    """One CFG + DDPM step of F frames (``sched``: a ``d4d_ddpm_sched`` from ``DDPMTables.c_struct``, which carries the
    noise seed).  ``noise`` [(cfg?2:1)*F,4,h,w]; ``frame_ids`` int64 [F]: each frame's index in its task.  Returns (new
    latents, advanced timestep indices)."""
    _bf16c(noise, "noise"), _bf16c(latents, "latents"), _bf16c(cond_mask, "cond_mask")
    F, _, h, w = latents.shape
    for name, t in (("timestep_indices", timestep_indices), ("frame_ids", frame_ids)):
        if t.dtype != torch.int64 or not t.is_cuda or not t.is_contiguous() or t.numel() != F:
            raise ValueError(f"{name} must be a contiguous CUDA int64 [F] tensor")
    out = torch.empty_like(latents)
    ti_out = torch.empty_like(timestep_indices)
    check(lib().d4d_cfg_ddpm_step(_p(noise), _p(latents), _p(cond_mask), _p(timestep_indices), _p(ti_out), _p(frame_ids),
                                  C.byref(sched), float(guidance_scale), int(cfg), F, h, w, _p(out), _stream()),
          "d4d_cfg_ddpm_step")
    return out, ti_out


def ddpm_noise(seed: int, frame_ids: torch.Tensor, timestep_indices: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """The DDPM step's noise z of frames ``frame_ids`` (int64 [F]) at ``timestep_indices`` (int64 [F]) for the task
    ``seed``, rounded once to fp32: [F, 4, h, w]."""
    F = frame_ids.numel()
    for name, t in (("frame_ids", frame_ids), ("timestep_indices", timestep_indices)):
        if t.dtype != torch.int64 or not t.is_cuda or not t.is_contiguous() or t.numel() != F:
            raise ValueError(f"{name} must be a contiguous CUDA int64 [F] tensor")
    out = torch.empty(F, 4, h, w, dtype=torch.float32, device=frame_ids.device)
    check(lib().d4d_op_ddpm_noise(int(seed) & 0xFFFFFFFFFFFFFFFF, _p(frame_ids), _p(timestep_indices), F, h, w, _p(out),
                                  _stream()), "d4d_op_ddpm_noise")
    return out
