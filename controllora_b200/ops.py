"""Thin Python wrappers over the C ABI.  Tensors are torch CUDA tensors used purely as device-memory handles."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib
from ._lib import GemmArgs, check

BF16 = torch.bfloat16


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else C.c_void_p(t.data_ptr())


def _req(t: torch.Tensor, dtype, name: str):
    if not t.is_cuda:
        raise _lib.CLError(f"{name}: controllora_b200 ops need CUDA tensors (no CPU fallback)")
    if t.dtype != dtype:
        raise _lib.CLError(f"{name}: expected {dtype}, got {t.dtype}")


def gemm(
    a: torch.Tensor,
    b: torch.Tensor,
    *,
    out: Optional[torch.Tensor] = None,
    bias: Optional[torch.Tensor] = None,
    row_bias: Optional[torch.Tensor] = None,
    rows_per_group: int = 0,
    residual: Optional[torch.Tensor] = None,
    ext: Optional[torch.Tensor] = None,
    lora_up: Optional[torch.Tensor] = None,
    lora_scale: float = 1.0,
    t_add: Optional[torch.Tensor] = None,
    t_out: Optional[torch.Tensor] = None,
    out_fp32: bool = False,
    conv_stride: int = 0,
    pad_lo: int = 1,
    block_n: int = 0,
) -> torch.Tensor:
    """D = epilogue(A @ B^T).  `a` is [M, K] bf16, or an NHWC image [n, H, W, C] when conv_stride in {1, 2}
    (3x3 implicit GEMM, `b` = [N, 9*C])."""
    _req(a, BF16, "a")
    _req(b, BF16, "b")
    args = GemmArgs()
    N, K = b.shape
    if conv_stride:
        n_img, H, W, Cc = a.shape
        assert a.is_contiguous()
        args.a_mode = 1 if conv_stride == 1 else 2
        args.n_img, args.H, args.W, args.C = n_img, H, W, Cc
        args.pad_lo = pad_lo
        M = n_img * (H // conv_stride) * (W // conv_stride)
        assert K == 9 * Cc
        out_shape = (n_img, H // conv_stride, W // conv_stride, N)
    else:
        assert a.dim() == 2 and a.stride(1) == 1 and a.shape[1] == K
        M = a.shape[0]
        args.a_mode = 0
        args.lda = a.stride(0)
        out_shape = (M, N)
    assert b.stride(1) == 1
    args.M, args.N, args.K = M, N, K
    args.a = _ptr(a)
    args.b = _ptr(b)
    args.ldb = b.stride(0)
    if out is None:
        out = torch.empty(out_shape, device=a.device, dtype=torch.float32 if out_fp32 else BF16)
    else:
        _req(out, torch.float32 if out_fp32 else BF16, "out")
    out2d = out.view(-1, N) if out.is_contiguous() else out
    assert out2d.dim() == 2 and out2d.stride(1) == 1 and out2d.shape[0] == M
    args.out = _ptr(out2d)
    args.ldd = out2d.stride(0)
    args.out_fp32 = 1 if out_fp32 else 0
    if bias is not None:
        _req(bias, torch.float32, "bias")
        args.bias = _ptr(bias)
    if row_bias is not None:
        _req(row_bias, torch.float32, "row_bias")
        assert row_bias.dim() == 2 and row_bias.stride(1) == 1 and row_bias.shape[-1] == N
        args.row_bias = _ptr(row_bias)
        args.rows_per_group = rows_per_group
        args.ld_row_bias = row_bias.stride(0)
    if residual is not None:
        _req(residual, BF16, "residual")
        r2 = residual.view(-1, N) if residual.is_contiguous() else residual
        assert r2.stride(1) == 1 and r2.shape[0] == M
        args.residual = _ptr(r2)
        args.ldr = r2.stride(0)
    if lora_up is not None:
        _req(lora_up, torch.float32, "lora_up")
        _req(ext, BF16, "ext")
        assert ext.shape == (16, K) and ext.stride(1) == 1
        assert lora_up.is_contiguous() and lora_up.shape[0] == N and lora_up.shape[1] in (4, 8)
        args.ext = _ptr(ext)
        args.ldb_ext = ext.stride(0)
        args.lora_up = _ptr(lora_up)
        args.lora_rp = lora_up.shape[1]
        args.lora_scale = float(lora_scale)
        if t_add is not None:
            _req(t_add, torch.float32, "t_add")
            assert t_add.is_contiguous() and t_add.shape == (M, lora_up.shape[1])
            args.t_add = _ptr(t_add)
        if t_out is not None:
            _req(t_out, torch.float32, "t_out")
            assert t_out.is_contiguous() and t_out.shape == (M, lora_up.shape[1])
            args.t_out = _ptr(t_out)
    args.block_n = block_n
    lib = _lib.lib()
    if lora_up is None and M <= 4096 and K >= 2048:
        # few output tiles, deep K: cut K across otherwise idle SMs (deterministic partial-tile sums, no atomics)
        splits = lib.cl_gemm_split_hint(C.byref(args))
        if splits > 1:
            ws = _split_ws(splits * M * N, a.device)
            args.split_k = splits
            args.split_ws = _ptr(ws)
    check(lib.cl_gemm(C.byref(args), _stream()), "cl_gemm")
    return out


_SPLIT_WS = {}
_WS_GRAVEYARD = []   # outgrown scratch buffers: a captured CUDA graph may have their addresses baked in, so they are kept
                     # alive for the process lifetime instead of going back to the caching allocator (a few MB each)


def _split_ws(numel: int, device) -> torch.Tensor:
    """fp32 scratch for split-K partial tiles, one growing buffer per device (stream-ordered re-use)."""
    buf = _SPLIT_WS.get(device)
    if buf is None or buf.numel() < numel:
        if buf is not None:
            _WS_GRAVEYARD.append(buf)
        buf = torch.empty(max(numel, 1 << 22), device=device, dtype=torch.float32)
        _SPLIT_WS[device] = buf
    return buf


def split_bf16_ext(down: torch.Tensor, k: int) -> torch.Tensor:
    """Pack LoRA-down rows (fp32 [r<=8, k]) into the [16, k] bf16 `ext` operand: rows j / j+8 = hi / lo split."""
    r = down.shape[0]
    assert r <= 8 and down.shape[1] == k
    ext = torch.zeros(16, k, device=down.device, dtype=BF16)
    hi = down.to(BF16)
    lo = (down - hi.float()).to(BF16)
    ext[:r] = hi
    ext[8 : 8 + r] = lo
    return ext


# ----------------------------------------------------------------------------------------------------------------
# generic helpers for the flat (non-struct) entry points
# ----------------------------------------------------------------------------------------------------------------
def _call(name: str, *args):
    fn = getattr(_lib.lib(), name)
    check(fn(*args, _stream()), name)


def _p(t):
    return C.c_void_p(0) if t is None else C.c_void_p(t.data_ptr())


def attention_fwd(q, k, v, heads: int, scale: float, out=None, need_lse=True):
    """q [B, Nq, H*d], k/v [B, Nk, H*d] bf16 (last dim contiguous, arbitrary row stride) -> o [B, Nq, H*d], lse [B,H,Nq]."""
    from ._lib import AttnFwdArgs

    _req(q, BF16, "q"); _req(k, BF16, "k"); _req(v, BF16, "v")
    B, Nq, HD = q.shape
    Nk = k.shape[1]
    d = HD // heads
    for t in (q, k, v):
        assert t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    if out is None:
        out = torch.empty(B, Nq, HD, device=q.device, dtype=BF16)
    lse = torch.empty(B, heads, Nq, device=q.device, dtype=torch.float32) if need_lse else None
    a = AttnFwdArgs()
    a.B, a.H, a.Nq, a.Nk, a.d = B, heads, Nq, Nk, d
    a.q, a.ldq = _ptr(q), q.stride(1)
    a.k, a.ldk = _ptr(k), k.stride(1)
    a.v, a.ldv = _ptr(v), v.stride(1)
    a.o, a.ldo = _ptr(out), out.stride(1)
    a.lse = _ptr(lse)
    a.scale = float(scale)
    check(_lib.lib().cl_attn_fwd(C.byref(a), _stream()), "cl_attn_fwd")
    return out, lse


def groupnorm_fwd(x, gamma, beta, G: int, eps: float, silu: bool, out=None):
    """x NHWC [n, H, W, C] (or [n, HW, C]) bf16 -> (y, stats[n, G, 2])"""
    _req(x, BF16, "x")
    n, C_ = x.shape[0], x.shape[-1]
    HW = x.numel() // (n * C_)
    assert x.is_contiguous()
    y = torch.empty_like(x) if out is None else out
    stats = torch.empty(n, G, 2, device=x.device, dtype=torch.float32)
    _call("cl_groupnorm_fwd", _p(x), _p(gamma), _p(beta), _p(y), _p(stats), n, HW, C_, G, C.c_float(eps), int(silu))
    return y, stats


def groupnorm_bwd(x, dy, gamma, beta, stats, G: int, silu: bool, dx=None, accumulate=False, dgamma=None, dbeta=None):
    n, C_ = x.shape[0], x.shape[-1]
    HW = x.numel() // (n * C_)
    assert x.is_contiguous() and dy.is_contiguous()
    if dx is None:
        dx = torch.empty_like(x)
        accumulate = False
    _call("cl_groupnorm_bwd", _p(x), _p(dy), _p(gamma), _p(beta), _p(stats), _p(dx), _p(dgamma), _p(dbeta),
          n, HW, C_, G, int(silu), int(accumulate))
    return dx


def layernorm_fwd(x, gamma, beta, eps: float = 1e-5):
    _req(x, BF16, "x")
    assert x.is_contiguous()
    C_ = x.shape[-1]
    T = x.numel() // C_
    y = torch.empty_like(x)
    stats = torch.empty(T, 2, device=x.device, dtype=torch.float32)
    _call("cl_layernorm_fwd", _p(x), _p(gamma), _p(beta), _p(y), _p(stats), T, C_, C.c_float(eps))
    return y, stats


def layernorm_bwd(x, dy, gamma, stats, dx=None, accumulate=False):
    C_ = x.shape[-1]
    T = x.numel() // C_
    assert x.is_contiguous() and dy.is_contiguous()
    if dx is None:
        dx = torch.empty_like(x)
        accumulate = False
    _call("cl_layernorm_bwd", _p(x), _p(dy), _p(gamma), _p(stats), _p(dx), T, C_, int(accumulate))
    return dx


def geglu_fwd(p):
    F2 = p.shape[-1]
    T = p.numel() // F2
    out = torch.empty(*p.shape[:-1], F2 // 2, device=p.device, dtype=BF16)
    _call("cl_geglu_fwd", _p(p), _p(out), C.c_int64(T), F2 // 2)
    return out


def geglu_bwd(p, dout):
    F2 = p.shape[-1]
    T = p.numel() // F2
    dp = torch.empty_like(p)
    _call("cl_geglu_bwd", _p(p), _p(dout), _p(dp), C.c_int64(T), F2 // 2)
    return dp


def add(a, b, out=None):
    assert a.is_contiguous() and b.is_contiguous() and a.shape == b.shape
    out = torch.empty_like(a) if out is None else out
    _call("cl_add", _p(a), _p(b), _p(out), C.c_int64(a.numel()))
    return out


def upsample2x_fwd(x):
    n, H, W, C_ = x.shape
    y = torch.empty(n, 2 * H, 2 * W, C_, device=x.device, dtype=BF16)
    _call("cl_upsample2x_fwd", _p(x), _p(y), n, H, W, C_)
    return y


def upsample2x_bwd(dy, dx=None, accumulate=False):
    n, H2, W2, C_ = dy.shape
    if dx is None:
        dx = torch.empty(n, H2 // 2, W2 // 2, C_, device=dy.device, dtype=BF16)
        accumulate = False
    _call("cl_upsample2x_bwd", _p(dy), _p(dx), n, H2 // 2, W2 // 2, C_, int(accumulate))
    return dx


def zero_insert2x(x, off: int):
    n, H, W, C_ = x.shape
    y = torch.empty(n, 2 * H, 2 * W, C_, device=x.device, dtype=BF16)
    _call("cl_zero_insert2x", _p(x), _p(y), n, H, W, C_, off)
    return y


def concat_channels(a, b):
    Ca, Cb = a.shape[-1], b.shape[-1]
    M = a.numel() // Ca
    out = torch.empty(*a.shape[:-1], Ca + Cb, device=a.device, dtype=BF16)
    _call("cl_concat_channels", _p(a), _p(b), _p(out), C.c_int64(M), Ca, Cb)
    return out


def slice_channels(src, c_off: int, Cd: int, dst=None, accumulate=False):
    Cs = src.shape[-1]
    M = src.numel() // Cs
    if dst is None:
        dst = torch.empty(*src.shape[:-1], Cd, device=src.device, dtype=BF16)
        accumulate = False
    _call("cl_slice_channels", _p(src), _p(dst), C.c_int64(M), Cs, c_off, Cd, int(accumulate))
    return dst


def nchw_to_nhwc(x):
    n, C_, H, W = x.shape
    assert x.is_contiguous() and x.dtype in (torch.float32, BF16)
    y = torch.empty(n, H, W, C_, device=x.device, dtype=BF16)
    _call("cl_nchw_to_nhwc", _p(x), int(x.dtype == torch.float32), _p(y), n, C_, H * W)
    return y


def nhwc_to_nchw_f32(x, out=None, accumulate=False):
    n, H, W, C_ = x.shape
    if out is None:
        out = torch.empty(n, C_, H, W, device=x.device, dtype=torch.float32)
        accumulate = False
    _call("cl_nhwc_to_nchw_f32", _p(x), _p(out), n, C_, H * W, int(accumulate))
    return out


def f32_to_bf16(x):
    y = torch.empty(x.shape, device=x.device, dtype=BF16)
    _call("cl_f32_to_bf16", _p(x), _p(y), C.c_int64(x.numel()))
    return y


def conv_in(x, w, bias, cout: int):
    """x NCHW fp32 [n, Cin, H, W]; w bf16 [Cout, 3, 3, Cin] -> NHWC bf16"""
    n, Cin, H, W = x.shape
    _req(x, torch.float32, "x")
    y = torch.empty(n, H, W, cout, device=x.device, dtype=BF16)
    _call("cl_conv_in", _p(x.contiguous()), _p(w), _p(bias), _p(y), n, Cin, H, W, cout)
    return y


def conv_out(x, w, bias):
    n, H, W, C_ = x.shape
    y = torch.empty(n, 4, H, W, device=x.device, dtype=torch.float32)
    _call("cl_conv_out", _p(x), _p(w), _p(bias), _p(y), n, H, W, C_, 4)
    return y


def conv_out_bwd(dy, w, C_: int):
    n, _, H, W = dy.shape
    dx = torch.empty(n, H, W, C_, device=dy.device, dtype=BF16)
    _call("cl_conv_out_bwd", _p(dy.contiguous()), _p(w), _p(dx), n, H, W, C_, 4)
    return dx


def timestep_embedding(t, dim: int):
    t = t.to(torch.float32).contiguous()
    out = torch.empty(t.shape[0], dim, device=t.device, dtype=torch.float32)
    _call("cl_timestep_embedding", _p(t), _p(out), t.shape[0], dim)
    return out


def small_linear(x, w, bias, silu_in=False, silu_out=False):
    Bt, K = x.shape
    N = w.shape[0]
    out = torch.empty(Bt, N, device=x.device, dtype=torch.float32)
    _call("cl_small_linear", _p(x), _p(w), _p(bias), _p(out), Bt, N, K, int(silu_in), int(silu_out))
    return out


def mse_loss(pred, target, gscale: float = 1.0, need_grad=True, out=None):
    """loss = mean((pred - target)^2);  dpred = gscale * 2 (pred - target) / n  (written into `out` when given)."""
    assert pred.is_contiguous() and target.is_contiguous() and (out is None or out.is_contiguous())
    loss = torch.empty(1, device=pred.device, dtype=torch.float32)
    dpred = out if out is not None else (torch.empty_like(pred) if need_grad else None)
    _call("cl_mse_loss", _p(pred), _p(target), _p(loss), _p(dpred), C.c_int64(pred.numel()), C.c_float(gscale))
    return loss, dpred


def add_noise(x0, sqrt_ac, sqrt_1mac, step_counter, seed: int, v_prediction: bool = False, out=None):
    """Device-side `randn_like` + `randint` + `add_noise` + target selection (train_text_to_image_control_lora.py:757-779).
    x0 [B, ...] fp32; sqrt_ac / sqrt_1mac fp32 [T] device tables; step_counter: int64 [1] device tensor (advanced by one).
    Returns (noisy, target, timesteps fp32 [B])."""
    _req(x0, torch.float32, "x0")
    assert x0.is_contiguous() and step_counter.dtype == torch.int64 and step_counter.is_cuda
    B = x0.shape[0]
    per = x0.numel() // B
    noisy, target, ts = out if out is not None else (torch.empty_like(x0), torch.empty_like(x0),
                                                     torch.empty(B, device=x0.device, dtype=torch.float32))
    _call("cl_add_noise", _p(x0), _p(sqrt_ac), _p(sqrt_1mac), _p(step_counter), C.c_uint64(seed & (2**64 - 1)), sqrt_ac.numel(),
          int(v_prediction), _p(noisy), _p(target), _p(ts), B, per)
    return noisy, target, ts


def attention_bwd(q, k, v, o, d_o, lse, heads: int, scale: float, need_dq=True, need_dkv=True, dq=None, dk=None, dv=None):
    from ._lib import AttnBwdArgs

    B, Nq, HD = q.shape
    Nk = k.shape[1]
    d = HD // heads
    for t in (q, k, v, o, d_o):
        assert t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    delta = torch.empty(B, heads, Nq, device=q.device, dtype=torch.float32)
    if need_dq and dq is None:
        dq = torch.empty(B, Nq, HD, device=q.device, dtype=BF16)
    if need_dkv and dk is None:
        dk = torch.empty(B, Nk, HD, device=q.device, dtype=BF16)
        dv = torch.empty(B, Nk, HD, device=q.device, dtype=BF16)
    a = AttnBwdArgs()
    a.B, a.H, a.Nq, a.Nk, a.d = B, heads, Nq, Nk, d
    a.q, a.ldq = _ptr(q), q.stride(1)
    a.k, a.ldk = _ptr(k), k.stride(1)
    a.v, a.ldv = _ptr(v), v.stride(1)
    a.o, a.ldo = _ptr(o), o.stride(1)
    a.d_o, a.lddo = _ptr(d_o), d_o.stride(1)
    a.lse, a.delta = _ptr(lse), _ptr(delta)
    if need_dq:
        a.dq, a.lddq = _ptr(dq), dq.stride(1)
    if need_dkv:
        a.dk, a.lddk = _ptr(dk), dk.stride(1)
        a.dv, a.lddv = _ptr(dv), dv.stride(1)
    a.scale = float(scale)
    check(_lib.lib().cl_attn_bwd(C.byref(a), _stream()), "cl_attn_bwd")
    return dq, dk, dv


class PackPlan:
    """Device-resident descriptor table for cl_lora_pack_batch (built once; re-run every step)."""

    def __init__(self, device):
        self.device = device
        self.descs = []
        self.max_elems = 1
        self._dev = None
        self._keep = []
        self._unscaled = []      # descriptor indices whose `mul` follows 1/scale (set_unscaled_mul)
        self._unscaled_mul = 1.0

    def add(self, src: torch.Tensor, dst: torch.Tensor, kind: int, r: int, K: int, s_j: int, s_k: int, ld: int, row_off: int,
            unscaled: bool = False):
        from ._lib import PackDesc

        # bounds of the packed operand (an out-of-range descriptor would be a silent out-of-bounds device write)
        if kind == 0 and not (0 <= row_off and row_off + r <= 8 and dst.shape[0] == 16 and K <= dst.shape[1]):
            raise ValueError(f"PackPlan: ext rows [{row_off}, {row_off + r}) x {K} do not fit the 8+8 hi/lo rows of {tuple(dst.shape)}")
        if kind == 1 and not (0 <= row_off and row_off + r <= dst.shape[1] and K <= dst.shape[0]):
            raise ValueError(f"PackPlan: table columns [{row_off}, {row_off + r}) do not fit {tuple(dst.shape)}")
        if kind == 2 and not (0 <= row_off and row_off + r <= 8 and 8 + row_off + r <= dst.shape[1] and K <= dst.shape[0]):
            raise ValueError(f"PackPlan: transposed hi/lo columns [{row_off}, {row_off + r}) do not fit {tuple(dst.shape)}")
        d = PackDesc()
        d.src, d.dst = src.data_ptr(), dst.data_ptr()
        d.kind, d.r, d.K, d.s_j, d.s_k, d.ld, d.row_off = kind, r, K, s_j, s_k, ld, row_off
        d.mul = self._unscaled_mul if unscaled else 1.0
        if unscaled:
            self._unscaled.append(len(self.descs))
        self.descs.append(d)
        self._keep.append((src, dst))
        self.max_elems = max(self.max_elems, r * K)
        self._dev = None

    def set_unscaled_mul(self, mul: float) -> None:
        """Adapters flagged `unscaled` (stacked pre/post value adapters, models.py:260,265,397,402: their delta is added
        WITHOUT `scale`) are packed with mul = 1/scale so that the fused epilogue's common `scale` cancels."""
        if mul != self._unscaled_mul:
            self._unscaled_mul = mul
            for i in self._unscaled:
                self.descs[i].mul = mul
            if self._unscaled:
                self._dev = None

    def add_ext(self, down_like: torch.Tensor, ext: torch.Tensor, row_off: int = 0, transposed: bool = False, unscaled: bool = False):
        """ext rows <- rows of `down_like` ([r, K]); transposed=True reads a [K, r] matrix (e.g. up.weight) instead."""
        if transposed:
            K, r = down_like.shape
            self.add(down_like, ext, 0, r, K, down_like.stride(1), down_like.stride(0), ext.stride(0), row_off, unscaled)
        else:
            r, K = down_like.shape
            self.add(down_like, ext, 0, r, K, down_like.stride(0), down_like.stride(1), ext.stride(0), row_off, unscaled)

    def add_table(self, up_like: torch.Tensor, table: torch.Tensor, col_off: int = 0, transposed: bool = False, unscaled: bool = False):
        """table[n, col_off + j] <- up_like[n, j] ([N, r]); transposed=True reads a [r, N] matrix (down.weight)."""
        if transposed:
            r, N = up_like.shape
            self.add(up_like, table, 1, r, N, up_like.stride(0), up_like.stride(1), table.stride(0), col_off, unscaled)
        else:
            N, r = up_like.shape
            self.add(up_like, table, 1, r, N, up_like.stride(1), up_like.stride(0), table.stride(0), col_off, unscaled)

    def run(self):
        from ._lib import PackDesc

        if not self.descs:
            return
        if self._dev is None:
            arr = (PackDesc * len(self.descs))(*self.descs)
            raw = bytes(arr)
            host = torch.frombuffer(bytearray(raw), dtype=torch.uint8)
            self._dev = host.to(self.device)
        _call("cl_lora_pack_batch", C.c_void_p(self._dev.data_ptr()), len(self.descs), self.max_elems)


def skinny_atb(a, r: int, b, out, so_j: int, so_c: int, alpha: float):
    """out[j*so_j + c*so_c] += alpha * sum_m a[m, j] * b[m, c];  a fp32 [M, lda], b bf16 [M, C]"""
    M = a.shape[0]
    b2 = b.view(-1, b.shape[-1]) if b.is_contiguous() else b
    assert b2.shape[0] == M and b2.stride(1) == 1
    _call("cl_skinny_atb", _p(a), a.stride(0), r, _p(b2), C.c_int64(b2.stride(0)), _p(out), C.c_int64(so_j), C.c_int64(so_c),
          C.c_float(alpha), M, b2.shape[1])


def rowdot(a, u):
    """e[m, j] = sum_n a[m, n] * u[n, j];  a bf16 [M, N], u fp32 [N, rp]"""
    a2 = a.view(-1, a.shape[-1]) if a.is_contiguous() else a
    M, N = a2.shape
    rp = u.shape[1]
    e = torch.empty(M, rp, device=a.device, dtype=torch.float32)
    _call("cl_rowdot", _p(a2), C.c_int64(a2.stride(0)), _p(u), rp, _p(e), M, N)
    return e


def rowmat(a, w, sw_i: int, sw_j: int, I: int, J: int, alpha: float, out, ldo: int, out_mode=0, col_off=0, lo_off=0, accumulate=False):
    M = a.shape[0]
    _call("cl_rowmat", _p(a), a.stride(0), _p(w), sw_i, sw_j, I, J, C.c_float(alpha), _p(out), ldo, out_mode, col_off, lo_off,
          int(accumulate), M)


def skinny_small(a, I: int, b, J: int, out, alpha: float):
    _call("cl_skinny_small", _p(a), a.stride(0), I, _p(b), b.stride(0), J, _p(out), C.c_float(alpha), a.shape[0])


def small_matmul(a, sa_i, sa_j, b, sb_j, sb_k, out, so_i, so_k, I, J, K, alpha=1.0, accumulate=False):
    _call("cl_small_matmul", _p(a), C.c_int64(sa_i), C.c_int64(sa_j), _p(b), C.c_int64(sb_j), C.c_int64(sb_k), _p(out),
          C.c_int64(so_i), C.c_int64(so_k), I, J, K, C.c_float(alpha), int(accumulate))


def sumsq(x, out):
    _call("cl_sumsq", _p(x), C.c_int64(x.numel()), _p(out))


def adamw(p, g, m, v, lr, beta1, beta2, eps, wd, step, gnorm_sq=None, max_norm=0.0, grad_scale=1.0, zero_grad=True):
    _call("cl_adamw", _p(p), _p(g), _p(m), _p(v), C.c_int64(p.numel()), C.c_float(lr), C.c_float(beta1), C.c_float(beta2),
          C.c_float(eps), C.c_float(wd), int(step), _p(gnorm_sq), C.c_float(max_norm), C.c_float(grad_scale), int(zero_grad))


def step_begin(gnorm_sq, step_dev):
    _call("cl_step_begin", _p(gnorm_sq), _p(step_dev))


def adamw_dev(p, g, m, v, lr, beta1, beta2, eps, wd, step_dev, gnorm_sq=None, max_norm=0.0, grad_scale=1.0, zero_grad=True):
    """AdamW whose bias corrections come from the device-side step counter `step_dev` (int64 [1], advanced by step_begin)."""
    _call("cl_adamw_dev", _p(p), _p(g), _p(m), _p(v), C.c_int64(p.numel()), C.c_float(lr), C.c_float(beta1), C.c_float(beta2),
          C.c_float(eps), C.c_float(wd), _p(step_dev), _p(gnorm_sq), C.c_float(max_norm), C.c_float(grad_scale), int(zero_grad))


def hilo_combine(src, nb: int):
    M = src.shape[0]
    dst = torch.empty(M, 8 * nb, device=src.device, dtype=torch.float32)
    _call("cl_hilo_combine", _p(src), _p(dst), C.c_int64(M), nb)
    return dst


def rank_update(x, t, tab, alpha: float, out=None):
    """out = x + alpha * t[:, :rp] @ tab^T ; x bf16 [M, C], t fp32 [M, ldt], tab fp32 [C, rp]"""
    Cc = x.shape[-1]
    M = x.numel() // Cc
    out = torch.empty_like(x) if out is None else out
    _call("cl_rank_update", _p(x), _p(t), t.stride(0), _p(tab), tab.shape[1], C.c_float(alpha), _p(out), C.c_int64(M), Cc)
    return out


def v2_inject_fwd(x, th16, uc, rc: int, tab, alpha: float):
    """t = hilo(th16) + uc;  out = x + alpha * t[:, :4] @ tab^T.  x bf16 [..., C], th16 fp32 [M, 16], uc fp32 [M, >=rc] view,
    tab fp32 [C, 4].  Returns (out, t [M, 8])."""
    Cc = x.shape[-1]
    M = x.numel() // Cc
    assert x.is_contiguous() and th16.is_contiguous() and th16.shape == (M, 16) and tab.shape == (Cc, 4)
    assert uc is None or uc.shape[0] == M, "control product rows != hidden-state rows"
    out = torch.empty_like(x)
    t = torch.empty(M, 8, device=x.device, dtype=torch.float32)
    ldu = 0 if uc is None else uc.stride(0)
    _call("cl_v2_inject_fwd", _p(x), _p(th16), _p(uc), ldu, rc, _p(tab), C.c_float(alpha), _p(out), _p(t), C.c_int64(M), Cc)
    return out, t


def v2_inject_bwd(dy, up_tab, down_tab, alpha: float, need_dh: bool):
    """dt [M, 4] = dy @ up_tab;  dh = dy + alpha * dt @ down_tab^T (None unless need_dh)."""
    Cc = dy.shape[-1]
    M = dy.numel() // Cc
    assert dy.is_contiguous()
    dt = torch.empty(M, 4, device=dy.device, dtype=torch.float32)
    dh = torch.empty_like(dy) if need_dh else None
    _call("cl_v2_inject_bwd", _p(dy), _p(up_tab), _p(down_tab), C.c_float(alpha), _p(dt), _p(dh), M, Cc)
    return dt, dh


def rank4_project_update(x, proj_tab, upd_tab, uc, rc: int, alpha: float):
    """t [M, 4] = x @ proj_tab (+ uc[:, :rc]);  y = x + alpha * t @ upd_tab^T.  Tables fp32 [C, 4].  Returns (y, t)."""
    Cc = x.shape[-1]
    M = x.numel() // Cc
    assert x.is_contiguous()
    if uc is not None and uc.shape[0] != M:
        raise ValueError(f"control states cover {uc.shape[0]} tokens but the hidden states have {M}: inject control states with the UNet's "
                         f"batch size (e.g. control_lora(torch.cat([guide] * 2)) under classifier-free guidance)")
    t = torch.empty(M, 4, device=x.device, dtype=torch.float32)
    y = torch.empty_like(x)
    ldu = 0 if uc is None else uc.stride(0)
    _call("cl_rank4_project_update", _p(x), _p(proj_tab), _p(upd_tab), _p(uc), ldu, rc, C.c_float(alpha), _p(t), _p(y), M, Cc)
    return y, t


def conv_wgrad(dy, x, dw, ksize: int, stride: int = 1, pad_lo: int = 1, alpha: float = 1.0):
    """dw (fp32 [Cout, Cin, k, k], accumulated) += alpha * dY^T (*) X ; dy NHWC [n,Ho,Wo,Cout], x NHWC [n,H,W,Cin]"""
    n, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    assert dw.is_contiguous() and dw.dtype == torch.float32
    _call("cl_conv_wgrad", _p(dy), _p(x), _p(dw), n, H, W, Cin, Cout, ksize, stride, pad_lo, C.c_float(alpha))


def conv_weight_prep(w, wf, wd=None):
    Cout, Cin, k, _ = w.shape
    _call("cl_conv_weight_prep", _p(w), _p(wf), _p(wd), Cout, Cin, k)


def colsum(x, out, alpha: float = 1.0):
    Cc = x.shape[-1]
    M = x.numel() // Cc
    _call("cl_colsum", _p(x), _p(out), C.c_int64(M), Cc, C.c_float(alpha))


def conv_in_wgrad(x, dy, dw):
    n, Cin, H, W = x.shape
    _call("cl_conv_in_wgrad", _p(x), _p(dy), _p(dw), n, Cin, H, W, dy.shape[-1])


def cfg_ddim_step(eps2, latents, guidance, a_t, a_prev):
    """In-place DDIM (eta=0) update of `latents` [B,4,h,w] fp32 from eps2 [2B,4,h,w] = [uncond | cond]."""
    n_half = latents.numel()
    assert eps2.numel() == 2 * n_half and eps2.is_contiguous() and latents.is_contiguous()
    _call("cl_cfg_ddim_step", _p(eps2), _p(latents), C.c_int64(n_half), C.c_float(guidance), C.c_float(a_t ** 0.5),
          C.c_float((1 - a_t) ** 0.5), C.c_float(a_prev ** 0.5), C.c_float((1 - a_prev) ** 0.5))


def cfg_dpmpp_step(eps2, latents, x0_prev, guidance, alpha_s, sigma_s, c_x, c_m0, c_m1):
    """In-place DPM-Solver++(2M) update of `latents` (and of the stored x0 prediction) from eps2 [2B,...] = [uncond | cond]."""
    _req(eps2, torch.float32, "eps2")
    _req(latents, torch.float32, "latents")
    _req(x0_prev, torch.float32, "x0_prev")
    assert eps2.is_contiguous() and latents.is_contiguous() and x0_prev.is_contiguous()
    assert eps2.numel() == 2 * latents.numel() == 2 * x0_prev.numel()
    _call("cl_cfg_dpmpp_step", _p(eps2), _p(latents), _p(x0_prev), C.c_int64(latents.numel()), C.c_float(guidance),
          C.c_float(alpha_s), C.c_float(sigma_s), C.c_float(c_x), C.c_float(c_m0), C.c_float(c_m1))


def softmax_rows(s, scale: float):
    """p = softmax(scale * s, dim=-1) as bf16; s fp32 [R, C] contiguous (the VAE's one-head attention scores)."""
    _req(s, torch.float32, "s")
    assert s.dim() == 2 and s.is_contiguous()
    p = torch.empty(s.shape, device=s.device, dtype=BF16)
    _call("cl_softmax_rows", _p(s), _p(p), s.shape[0], s.shape[1], C.c_float(scale))
    return p


def clip_embed(ids, tok, pos):
    """x[b, t] = tok[ids[b, t]] + pos[t] (bf16); ids int64 [B, T]."""
    _req(tok, BF16, "tok")
    _req(pos, BF16, "pos")
    assert ids.dtype == torch.int64 and ids.is_contiguous() and ids.dim() == 2
    B, T = ids.shape
    Cc = tok.shape[1]
    out = torch.empty(B, T, Cc, device=tok.device, dtype=BF16)
    _call("cl_clip_embed", _p(ids), _p(tok), _p(pos), _p(out), B * T, T, Cc, tok.shape[0])
    return out


def quick_gelu_(x):
    """in place: x * sigmoid(1.702 x) (bf16, numel % 8 == 0)."""
    _req(x, BF16, "x")
    assert x.is_contiguous()
    _call("cl_quick_gelu", _p(x), C.c_int64(x.numel()))
    return x


def causal_attention_small(qkv, B: int, T: int, heads: int, scale: float):
    """causal softmax(q k^T * scale) v of a short sequence; qkv [B*T, 3*C] bf16 (q | k | v) -> [B*T, C] bf16."""
    _req(qkv, BF16, "qkv")
    assert qkv.is_contiguous() and qkv.shape[0] == B * T and qkv.shape[1] % (3 * heads) == 0
    Cc = qkv.shape[1] // 3
    out = torch.empty(B * T, Cc, device=qkv.device, dtype=BF16)
    _call("cl_causal_attention_small", _p(qkv), _p(out), B, T, heads, Cc // heads, C.c_float(scale))
    return out


def channel_affine_nchw(x, mul: float, shift):
    """y[n, c] = mul * x[n, c] + shift[c] on NCHW fp32."""
    _req(x, torch.float32, "x")
    _req(shift, torch.float32, "shift")
    n, Cc = x.shape[0], x.shape[1]
    y = torch.empty_like(x)
    _call("cl_channel_affine_nchw", _p(x), _p(y), _p(shift), C.c_float(mul), n, Cc, C.c_int64(x.numel() // (n * Cc)))
    return y


def cast_matrix(src, I: int, J: int, s_i: int, s_j: int, alpha: float = 1.0, out=None):
    """out[i, j] = bf16(alpha * src.flat[i*s_i + j*s_j]) for a strided (sliced / transposed) view of an fp32 master weight."""
    _req(src, torch.float32, "src")
    out = torch.empty(I, J, device=src.device, dtype=BF16) if out is None else out
    _call("cl_cast_matrix_bf16", _p(src), C.c_int64(s_i), C.c_int64(s_j), _p(out), C.c_int64(out.stride(0)), I, J, C.c_float(alpha))
    return out


def axpy_matrix(src, dst, alpha: float = 1.0):
    """dst[i, j] += alpha * src[i, j]; src fp32 contiguous [I, J], dst fp32 with row stride dst.stride(0), unit column stride."""
    _req(src, torch.float32, "src")
    _req(dst, torch.float32, "dst")
    I, J = src.shape[0], src.numel() // src.shape[0]
    assert src.is_contiguous() and dst.stride(-1) == 1 and dst.shape[0] == I
    _call("cl_axpy_matrix_f32", _p(src), _p(dst), C.c_int64(dst.stride(0)), I, J, C.c_float(alpha))


def sampler_prep(latents, x2, tt, ts_table, step_ctr):
    n_half = latents.numel()
    assert x2.numel() == 2 * n_half and latents.is_contiguous() and x2.is_contiguous() and step_ctr.dtype == torch.int64
    _call("cl_sampler_prep", _p(latents), _p(x2), _p(tt), _p(ts_table), _p(step_ctr), C.c_int64(n_half), tt.numel())


def cfg_solver_step_dev(eps2, latents, x0_prev, coef, step_ctr, guidance: float, kind: int):
    """CFG + (kind 0: DDIM | kind 1: DPM-Solver++(2M)) update with the step's coefficients read from coef[*step_ctr]; advances
    the device step counter.  eps2 [2B, ...] fp32 = [uncond | cond]."""
    _req(eps2, torch.float32, "eps2")
    _req(latents, torch.float32, "latents")
    assert eps2.is_contiguous() and latents.is_contiguous() and eps2.numel() == 2 * latents.numel()
    assert coef.dtype == torch.float32 and coef.is_contiguous() and coef.shape[1] == 8 and step_ctr.dtype == torch.int64
    _call("cl_cfg_solver_step_dev", _p(eps2), _p(latents), _p(x0_prev), _p(coef), _p(step_ctr), C.c_int64(latents.numel()),
          C.c_float(guidance), int(kind))


class SkinnyQueue:
    """Collects the rank-r gradient reductions (dA / dB of every LoRA adapter) and issues them CL_SKINNY_MAX at a time
    through cl_skinny_atb_batch.  The queue keeps the operand tensors alive until the launch is enqueued."""

    def __init__(self):
        from ._lib import SKINNY_MAX, SkinnyDesc

        self._Desc, self._max = SkinnyDesc, SKINNY_MAX
        self.descs, self.keep = [], []

    def add(self, a, r: int, b, out, so_j: int, so_c: int, alpha: float):
        b2 = b.view(-1, b.shape[-1]) if b.is_contiguous() else b
        assert b2.stride(1) == 1 and b2.shape[0] == a.shape[0]
        d = self._Desc()
        d.a, d.lda, d.r = a.data_ptr(), a.stride(0), r
        d.b, d.ldb = b2.data_ptr(), b2.stride(0)
        d.out, d.so_j, d.so_c = out.data_ptr(), so_j, so_c
        d.alpha, d.M, d.C = float(alpha), b2.shape[0], b2.shape[1]
        self.descs.append(d)
        self.keep.append((a, b, out))
        if len(self.descs) >= self._max:
            self.flush()

    def flush(self):
        if not self.descs:
            return
        arr = (self._Desc * len(self.descs))(*self.descs)
        _call("cl_skinny_atb_batch", arr, len(self.descs))
        self.descs, self.keep = [], []


SKINNY = SkinnyQueue()


def canny(images, thresholds, *, edges=None, guide=None, pixels=None):
    """cv2.Canny per image (aperture 3, L2gradient=False, bit for bit) on a uint8 NHWC batch [B, H, W, C], C = 1 or 3.
    thresholds: fp32 [B, 2] (lo, hi) on the device, read by the kernel (a captured graph replays with new values).  Fills
    any of: edges uint8 [B, H, W] (0 / 255), guide fp32 [B, 3, H, W] (+-1), pixels fp32 [B, 3, H, W] = img / 127.5 - 1
    (C = 3 only).  Returns (edges, guide, pixels)."""
    _req(images, torch.uint8, "images")
    _req(thresholds, torch.float32, "thresholds")
    if images.dim() != 4 or not images.is_contiguous():
        raise _lib.CLError(f"images: expected a contiguous [B, H, W, C] tensor, got shape {tuple(images.shape)}")
    B, H, W, Cc = images.shape
    if thresholds.shape != (B, 2) or not thresholds.is_contiguous():
        raise _lib.CLError(f"thresholds: expected a contiguous [{B}, 2] tensor, got shape {tuple(thresholds.shape)}")
    for name, t, dtype, shape in (("edges", edges, torch.uint8, (B, H, W)), ("guide", guide, torch.float32, (B, 3, H, W)),
                                  ("pixels", pixels, torch.float32, (B, 3, H, W))):
        if t is None:
            continue
        _req(t, dtype, name)
        if tuple(t.shape) != shape or not t.is_contiguous():
            raise _lib.CLError(f"{name}: expected a contiguous {shape} tensor, got shape {tuple(t.shape)}")
        if t.device != images.device:
            raise _lib.CLError(f"{name}: on {t.device}, images on {images.device}")
    if thresholds.device != images.device:
        raise _lib.CLError(f"thresholds: on {thresholds.device}, images on {images.device}")
    labels = torch.empty(B * H * W, device=images.device, dtype=torch.int32)
    check(_lib.lib().cl_canny(_ptr(images), B, H, W, Cc, _ptr(thresholds), _ptr(labels), _ptr(edges), _ptr(guide), _ptr(pixels),
                              _stream()), "cl_canny")
    return edges, guide, pixels
