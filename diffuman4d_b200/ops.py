"""Op-level Python wrappers over the C ABI (one hot-path kernel each).  torch is used only for device memory
and the current stream; all arithmetic happens in libd4d.so."""
from __future__ import annotations

from typing import Optional

import torch

from ._lib import check, lib


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _bf16c(t: torch.Tensor, name: str):
    if t.dtype != torch.bfloat16 or not t.is_cuda or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous CUDA bfloat16 tensor")


def gemm(a: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, *, a2: Optional[torch.Tensor] = None,
         rowvec: Optional[torch.Tensor] = None, rows_per_image: int = 0, residual: Optional[torch.Tensor] = None,
         geglu: bool = False, act: int = 0, out_scale: float = 1.0, block_n: int = 0) -> torch.Tensor:
    """out = act((a | a2) @ w.T + bias + rowvec[row // rows_per_image]) * out_scale + residual   (bf16, fp32 accumulate).
    With ``geglu`` the rows of ``w``/``bias`` must already be tile-interleaved (see ``interleave_geglu``);
    ``block_n`` = 0 picks the tile width, otherwise it must be a multiple of 16 that divides N."""
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
                            int(geglu), act, float(out_scale), block_n, _stream()), "d4d_op_gemm")
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
            block_n: int = 0) -> torch.Tensor:
    """3x3 / stride 1 / pad 1 conv on NHWC activations.  ``w_octi``: [Cout, 9, Cin] (tap = ky*3+kx)."""
    _bf16c(x_nhwc, "x"), _bf16c(w_octi, "w")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_octi.shape[0]
    out = torch.empty(n, H, W, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    check(lib().d4d_op_conv3x3(_p(x_nhwc), n, H, W, Cin, _p(w_octi), Cout, _p(bias), _p(rowvec),
                               0 if rowvec is None else rowvec.stride(0), _p(residual), act, _p(out), block_n,
                               _stream()), "d4d_op_conv3x3")
    return out


def conv_weight_to_octi(w_oihw: torch.Tensor) -> torch.Tensor:
    co, ci, kh, kw = w_oihw.shape
    return w_oihw.permute(0, 2, 3, 1).reshape(co, kh * kw, ci).contiguous()


def attention(qkv: torch.Tensor, batch: int, seq: int, heads: int, head_dim: int, scale: float) -> torch.Tensor:
    """qkv: [batch*seq, 3*heads*head_dim] (q | k | v column blocks, head-major inside each).  Returns [batch*seq, heads*head_dim]."""
    _bf16c(qkv, "qkv")
    C = heads * head_dim
    if qkv.shape != (batch * seq, 3 * C):
        raise ValueError("qkv shape")
    out = torch.empty(batch * seq, C, device=qkv.device, dtype=torch.bfloat16)
    base = qkv.data_ptr()
    check(lib().d4d_op_attention(base, base + 2 * C, base + 4 * C, qkv.stride(0), _p(out), C, batch, seq, heads,
                                 head_dim, float(scale), _stream()), "d4d_op_attention")
    return out


def groupnorm(x1: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, groups: int, eps: float, silu: bool,
              x2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """x1: [n_img, hw, C1] (+ x2 [n_img, hw, C2] virtually concatenated on channels) -> [n_img, hw, C1+C2]."""
    _bf16c(x1, "x1")
    n_img, hw, C1 = x1.shape
    C2 = 0 if x2 is None else x2.shape[2]
    out = torch.empty(n_img, hw, C1 + C2, device=x1.device, dtype=torch.bfloat16)
    check(lib().d4d_op_groupnorm(_p(x1), C1, _p(x2), C2, n_img, hw, groups, float(eps), _p(gamma), _p(beta),
                                 int(silu), _p(out), _stream()), "d4d_op_groupnorm")
    return out


def conv3x3_stride2(x_nhwc: torch.Tensor, w_octi: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """3x3 / stride 2 / pad 1 conv (Downsample2D) through a strided tensor map: [n,H,W,Cin] -> [n,H/2,W/2,Cout]."""
    _bf16c(x_nhwc, "x"), _bf16c(w_octi, "w")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_octi.shape[0]
    out = torch.empty(n, H // 2, W // 2, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    check(lib().d4d_op_conv_resample(_p(x_nhwc), n, H, W, Cin, _p(w_octi), Cout, _p(bias), 1, 0, 0, _p(out), _stream()),
          "d4d_op_conv_resample")
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
                       single_launch: bool = True) -> torch.Tensor:
    """nearest x2 upsample followed by a 3x3 / pad 1 conv (Upsample2D) as four sub-pixel phases on the low-res input."""
    _bf16c(x_nhwc, "x")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_oihw.shape[0]
    out = torch.empty(n, 2 * H, 2 * W, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    phases = upsample_phase_weights(w_oihw)
    if single_launch:
        wp = torch.stack(phases).contiguous()                                          # [4, Cout, 4, Cin]
        check(lib().d4d_op_conv_resample(_p(x_nhwc), n, H, W, Cin, _p(wp), Cout, _p(bias), 3, 0, 0, _p(out), _stream()),
              "d4d_op_conv_resample")
        return out
    for ph, wp in enumerate(phases):
        check(lib().d4d_op_conv_resample(_p(x_nhwc), n, H, W, Cin, _p(wp), Cout, _p(bias), 2, ph >> 1, ph & 1, _p(out),
                                         _stream()), "d4d_op_conv_resample")
    return out


def conv3x3_groupnorm(x_nhwc: torch.Tensor, w_octi: torch.Tensor, bias: Optional[torch.Tensor], gamma: torch.Tensor,
                      beta: torch.Tensor, groups: int, eps: float, silu: bool, residual: Optional[torch.Tensor] = None):
    """conv3x3 whose epilogue accumulates the GroupNorm statistics of its output + the GroupNorm(+SiLU) that consumes them
    (no statistics pass).  Returns (conv_out, gn_out), both [n, H, W, Cout]."""
    _bf16c(x_nhwc, "x"), _bf16c(w_octi, "w")
    n, H, W, Cin = x_nhwc.shape
    Cout = w_octi.shape[0]
    conv_out = torch.empty(n, H, W, Cout, device=x_nhwc.device, dtype=torch.bfloat16)
    gn_out = torch.empty_like(conv_out)
    check(lib().d4d_op_conv3x3_groupnorm(_p(x_nhwc), n, H, W, Cin, _p(w_octi), Cout, _p(bias), _p(residual), groups,
                                         float(eps), _p(gamma), _p(beta), int(silu), _p(conv_out), _p(gn_out), _stream()),
          "d4d_op_conv3x3_groupnorm")
    return conv_out, gn_out


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    _bf16c(x, "x")
    rows, C = x.shape
    out = torch.empty_like(x)
    check(lib().d4d_op_layernorm(_p(x), rows, C, float(eps), _p(gamma), _p(beta), _p(out), _stream()),
          "d4d_op_layernorm")
    return out
