"""ctypes binding of ``_slb200.so`` — the hand-written sm_90a kernels.

Every wrapper takes torch CUDA tensors (or raw device pointers), launches on the *current*
torch stream (so it composes with CUDA-graph capture) and raises on a non-zero status.
There is deliberately no fallback here: on a CUDA box a missing/unloadable library is an
error (``require()``), never a silent switch to torch ops.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import c_double, c_float, c_int, c_longlong, c_uint32, c_uint64, c_void_p
from typing import Sequence

import torch

from . import build as _build

_lib = None
LAUNCHES = 0            # number of kernels launched through this module (bench's gpu_launches)


class NativeError(RuntimeError):
    pass


def available() -> bool:
    return os.path.exists(_build.LIB)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_build.LIB):
            raise NativeError(f"{_build.LIB} missing: run `python -m split_learning_b200.ops.build`")
        _lib = ctypes.CDLL(_build.LIB)
        _lib.slb_error_string.restype = ctypes.c_char_p
    return _lib


_preloaded = set()


def preload(device=None) -> None:
    """Load every kernel of the library on ``device`` now (see slb_preload_* for why)."""
    d = torch.cuda.current_device() if device is None else (torch.device(device).index or 0)
    if d in _preloaded:
        return
    with torch.cuda.device(d):
        bad = (lib().slb_preload_gemm() + lib().slb_preload_fused() + lib().slb_preload_elementwise()
               + lib().slb_preload_transformer() + lib().slb_preload_allreduce() + lib().slb_preload_ticket()
               + lib().slb_preload_audio())
    if bad:
        raise NativeError(f"{bad} kernels failed to load (wrong GPU architecture? this library is sm_90a only)")
    _preloaded.add(d)


def require():
    """Fail loudly when CUDA is present but the kernel library is not."""
    if torch.cuda.is_available():
        lib()


def _p(t) -> c_void_p:
    if t is None:
        return c_void_p(0)
    if isinstance(t, int):
        return c_void_p(t)
    return c_void_p(t.data_ptr())


def _dt(t) -> c_int:
    """Activation dtype code of the C API: 0 = bf16, 1 = fp32 (tensors or raw ``DevPtr`` views of peer memory)."""
    if isinstance(t, torch.Tensor):
        return c_int(1 if t.dtype == torch.float32 else 0)
    return c_int(1 if getattr(t, "itemsize", 2) == 4 else 0)


def _stream() -> c_void_p:
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(code: int, what: str, n: int = 1):
    global LAUNCHES
    if code != 0:
        msg = ""
        if code <= -2000:
            msg = lib().slb_error_string(-(code + 2000)).decode()
        elif code <= -1000:
            msg = "cudaFuncSetAttribute: " + lib().slb_error_string(-(code + 1000)).decode()
        elif code <= -100:
            msg = f"cuTensorMapEncodeTiled CUresult={-(code + 100)}"
        raise NativeError(f"{what} failed with status {code} {msg}")
    LAUNCHES += n


# ------------------------------------------------------------------ tensor-core ops
_TUNING = None


def _tuning():
    """Measured (BLOCK_N, split-K) table written by tools/tune_conv.py (falls back to the heuristic when absent)."""
    global _TUNING
    if _TUNING is None:
        import json
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "conv_tuning.json")
        try:
            with open(path) as f:
                _TUNING = json.load(f)
        except (OSError, ValueError):
            _TUNING = {"conv": {}, "wgrad": {}}
    return _TUNING


def conv_tiling(M: int, N: int, Ca: int, target_ctas: int = 96, flip: int = 0, ke: int = 64):
    """(block_n, k_split) for the implicit-GEMM conv: these problems are latency- not FLOP-bound at microbatch 32,
    so spread every layer over ~all SMs — narrow N tiles first, then split K (fp32 vector red.add + finalize).
    A measured entry of ``conv_tuning.json`` for exactly this shape wins over the heuristic."""
    hit = _tuning().get("conv" if ke == 64 else "conv_f32", {}).get(f"{M},{N},{Ca},{flip}")
    if hit:
        return int(hit["bn"]), int(hit["ks"])
    m_tiles = (M + 127) // 128
    bn = 64
    for cand in (256, 128, 64):
        if N % cand == 0 and m_tiles * (N // cand) >= target_ctas:
            bn = cand
            break
    bn = min(bn, N)
    tiles = m_tiles * (N // bn)
    k_iters = 9 * (Ca // ke)
    k_split = 1
    if tiles < target_ctas:
        k_split = max(1, min((128 + tiles - 1) // tiles, k_iters // 4))
    return bn, k_split


def _ke(t) -> int:
    return 32 if _dt(t).value == 1 else 64


def _cap(acc) -> c_longlong:
    return c_longlong(0 if acc is None else acc.numel())


def conv_partial_floats(M: int, N: int, k_split: int) -> int:
    """Floats of the split-K partial buffer a conv / dgrad with in-kernel finalisation (``counters``) needs."""
    return M * N * k_split if k_split > 1 else 0


def conv3x3_fwd(x, w_bf16, y, bias=None, col_sum=None, col_sumsq=None, acc=None, tiling=None, counters=None):
    """x [B,H,W,Cin], w [Cout,3,3,Cin] -> y [B,H,W,Cout] (pre-BN) + optional BN sums; x / w / y all bf16 (wgmma bf16)
    or all fp32 (wgmma tf32).  ``acc`` enables split-K.  With ``counters`` it is an fp32 buffer of at least
    ``conv_partial_floats(M, Cout, k_split)`` floats (no zeroing needed): every K slice stores its partial tiles there and
    the last slice of a tile to arrive adds them in slice order and produces y and the sums.  Without ``counters`` it is a
    zeroed fp32 [M, Cout] accumulator and a finalize kernel produces y."""
    B, H, W, Cin = x.shape
    Cout = w_bf16.shape[0]
    bn, ks = tiling or conv_tiling(B * H * W, Cout, Cin, ke=_ke(x))
    if acc is None:
        ks = 1
    _check(lib().slb_conv3x3_igemm(_p(x), _p(w_bf16), _p(y), _p(bias), _p(col_sum), _p(col_sumsq), c_int(B), c_int(H),
                                   c_int(W), c_int(Cin), c_int(Cout), c_int(0), c_int(Cin), c_int(Cout), c_int(bn), c_int(ks),
                                   _p(acc), _cap(acc), _p(counters), _dt(x), _stream()), "conv3x3_fwd")
    if ks > 1 and counters is None:
        conv_finalize(acc, bias, y, col_sum, col_sumsq)


def conv3x3_dgrad(dy, w_bf16, dx, acc=None, tiling=None, counters=None, bn_stats=None, publish=None):
    """dy [B,H,W,Cout] bf16, w [Cout,3,3,Cin] bf16 -> dx [B,H,W,Cin] bf16.
    ``bn_stats``: (y, mean, invstd, gamma, beta, relu, pool, dgamma, dbeta) of the *upstream* ConvBlock (BN + ReLU
    [+ MaxPool2]) whose output gradient is dx: the epilogue then also reduces that block's BatchNorm-backward sums."""
    B, H, W, Cout = dy.shape
    Cin = w_bf16.shape[3]
    bn, ks = tiling or conv_tiling(B * H * W, Cin, Cout, flip=1, ke=_ke(dy))
    if _dt(dy).value == 1:
        bn = max(bn, 32)
    if acc is None:
        ks = 1
    if bn_stats is not None:
        if ks > 1 and counters is None:
            raise NativeError("conv3x3_dgrad(bn_stats=) needs in-kernel split-K finalisation (counters)")
        uy, mean, istd, gamma, beta, relu, pool, dgamma, dbeta = bn_stats
        _check(lib().slb_conv3x3_dgrad_bnstats(_p(dy), _p(w_bf16), _p(dx), c_int(B), c_int(H), c_int(W), c_int(Cout), c_int(Cin),
                                               c_int(Cin), c_int(Cout), c_int(bn), c_int(ks), _p(acc), _cap(acc), _p(counters), _p(uy),
                                               _p(mean), _p(istd), _p(gamma), _p(beta), c_int(int(relu)), c_int(int(pool)), _p(dbeta), _p(dgamma),
                                               _stream()), "conv3x3_dgrad_bnstats")
        return
    if publish is not None:
        # ``publish = (ticket, flag_ptr, seq)``: the kernel's last CTA releases the mailbox flag of the slot ``dx`` points into
        ticket, flag, seq = publish
        _check(lib().slb_conv3x3_igemm_pub(_p(dy), _p(w_bf16), _p(dx), _p(None), _p(None), _p(None), c_int(B), c_int(H), c_int(W),
                                           c_int(Cout), c_int(Cin), c_int(1), c_int(Cin), c_int(Cout), c_int(bn), c_int(ks),
                                           _p(acc), _cap(acc), _p(counters), _dt(dy), _p(ticket), _p(flag), _p(seq), _stream()),
               "conv3x3_dgrad_pub")
        return
    _check(lib().slb_conv3x3_igemm(_p(dy), _p(w_bf16), _p(dx), _p(None), _p(None), _p(None), c_int(B), c_int(H), c_int(W),
                                   c_int(Cout), c_int(Cin), c_int(1), c_int(Cin), c_int(Cout), c_int(bn), c_int(ks), _p(acc),
                                   _cap(acc), _p(counters), _dt(dy), _stream()), "conv3x3_dgrad")
    if ks > 1 and counters is None:
        conv_finalize(acc, None, dx, None, None)


def conv_finalize(acc, bias, y, col_sum, col_sumsq):
    C = y.shape[-1]
    P = y.numel() // C
    _check(lib().slb_conv_finalize(_p(acc), _p(bias), _p(y), _p(col_sum), _p(col_sumsq), c_longlong(P), c_int(C), _dt(y),
                                   _stream()), "conv_finalize")


def conv_pixel_box(H: int, W: int, pixels: int = 128, padded: bool = False):
    """(tb, th, tw, ragged) of a conv tile (``pixels`` = 128) or wgrad K step (64 bf16 / 32 fp32 pixels): the box the
    kernels load for an H x W map.  ragged 0 = consecutive pixels (power-of-two maps), 1 = padded power-of-two box
    (``padded=True`` forces it), -1 = no box (W > pixels)."""
    out = (c_int * 4)()
    lib().slb_conv_pixel_box(c_int(H), c_int(W), c_int(pixels), c_int(int(padded)), out)
    return tuple(out)


def conv3x3_wgrad(x, dy, dw_f32, k_split: int = 0, block_n: int = 0):
    """dw [Cout,3,3,Cin] fp32 (+)= x^T (*) dy.  Split-K slices accumulate with red.add (caller zeroes dw); a layer
    whose K fits one slice is written with plain stores."""
    B, H, W, Cin = x.shape
    Cout = dy.shape[3]
    if k_split == 0 and block_n == 0:
        hit = _tuning().get("wgrad" if _ke(x) == 64 else "wgrad_f32", {}).get(f"{B * H * W},{Cin},{Cout}")
        if hit:
            block_n, k_split = int(hit["bn"]), int(hit["ks"])
    _check(lib().slb_conv3x3_wgrad(_p(x), _p(dy), _p(dw_f32), c_int(B), c_int(H), c_int(W), c_int(Cin), c_int(Cout),
                                   c_int(k_split), c_int(block_n), _dt(x), _stream()), "conv3x3_wgrad")


EPI_ATOMIC, EPI_ATOMIC_T, EPI_STORE = 1, 2, 3


def gemm_bf16(A, Bm, out, M, N, K, a_mn, b_mn, lda, ldb, ldo, epi, k_split=1, block_n=32):
    _check(lib().slb_gemm_bf16(_p(A), _p(Bm), _p(out), c_int(M), c_int(N), c_int(K), c_int(a_mn), c_int(b_mn),
                               c_longlong(lda), c_longlong(ldb), c_longlong(ldo), c_int(epi), c_int(k_split),
                               c_int(block_n), _stream()), "gemm_bf16")


def linear_fwd(x, w_bf16, acc, k_split=4):
    """acc[b][out] (fp32, zeroed) += x[b][in] @ w[out][in]^T  — swap-AB: out on the MMA M axis."""
    Bn, K = x.shape
    out_f = w_bf16.shape[0]
    gemm_bf16(w_bf16, x, acc, out_f, Bn, K, 0, 0, w_bf16.stride(0), x.stride(0), acc.stride(0), EPI_ATOMIC_T, k_split, 32)


def linear_dgrad(dz, w_bf16, dacc, k_split=4):
    """dacc[b][in] (fp32, zeroed) += dz[b][out] @ w[out][in]."""
    Bn = dz.shape[0]
    out_f, in_f = w_bf16.shape
    gemm_bf16(w_bf16, dz, dacc, in_f, Bn, out_f, 1, 0, w_bf16.stride(0), dz.stride(0), dacc.stride(0), EPI_ATOMIC_T,
              k_split, 32)


def linear_wgrad(dz, x, dw_f32):
    """dw[out][in] (fp32) = dz[b][out]^T @ x[b][in]   (plain store)."""
    Bn, in_f = x.shape
    out_f = dw_f32.shape[0]
    gemm_bf16(dz, x, dw_f32, out_f, in_f, Bn, 1, 1, dz.stride(0), x.stride(0), dw_f32.stride(0), EPI_STORE, 1,
              256 if in_f >= 256 else 64)


_NUM_SMS = {}


def num_sms(device=None) -> int:
    d = torch.cuda.current_device() if device is None else torch.device(device).index or 0
    if d not in _NUM_SMS:
        _NUM_SMS[d] = torch.cuda.get_device_properties(d).multi_processor_count
    return _NUM_SMS[d]


def conv_bn_act_p2p(x, w_bf16, bias, gamma, beta, running_mean, running_var, nbt, save_mean, save_invstd, col_sum, col_sumsq,
                    y_opt, out, relu, pool, grid_bar, momentum=0.1, eps=1e-5, update_running=True, flag=None, seq=None,
                    hint=None):
    """Fused cut-tail forward: conv3x3 -> batch stats -> grid barrier -> BN+ReLU(+pool) out of shared memory -> store into
    ``out`` (local or peer mailbox slot) -> publish flag.  ``y_opt``: optional local copy of the pre-BN output."""
    B, H, W, Cin = x.shape
    Cout = w_bf16.shape[0]
    _check(lib().slb_conv_bn_act_p2p(_p(x), _p(w_bf16), _p(bias), _p(gamma), _p(beta), _p(running_mean), _p(running_var),
                                     _p(nbt), _p(save_mean), _p(save_invstd), _p(col_sum), _p(col_sumsq), _p(y_opt), _p(out),
                                     c_int(B), c_int(H), c_int(W), c_int(Cin), c_int(Cout), c_int(int(relu)), c_int(int(pool)),
                                     c_float(momentum), c_float(eps), c_int(int(update_running)), _p(grid_bar), _p(flag),
                                     _p(seq), _p(hint), c_int(num_sms(x.device)), _dt(x), _stream()), "conv_bn_act_p2p")


def fused_cut_supported(B, H, W, Cin, Cout, pool, ke: int = 64) -> bool:
    if Cin % ke or Cout % 64 or 128 % W:
        return False
    rows = 128 // W
    th = rows if rows <= H else H
    if pool and ((th & 1) or (H & 1) or (W & 1)):
        return False
    bn = 256 if Cout >= 256 else Cout
    total = ((B * H * W + 127) // 128) * (Cout // bn)
    grid = min(total, num_sms() - 4)                  # the persistent grid of slb_conv_bn_act_p2p
    return (total + grid - 1) // grid <= (2 if bn <= 128 else 1)   # accumulator tiles per CTA that fit in shared memory


# ------------------------------------------------------------------ memory-bound ops
def zero_(t, wait=None):
    """Zero a scratch tensor.  ``wait = (flag_ptr, expect_ctr, max_spins, status)``: the same launch also acquires a mailbox
    slot flag (``zero_wait_kernel``) — the first kernel of a program that consumes a slot."""
    if wait is not None:
        flag_ptr, expect_ctr, max_spins, status = wait
        _check(lib().slb_zero_wait(_p(t), c_longlong(t.numel() * t.element_size()), c_void_p(flag_ptr), _p(expect_ctr),
                                   c_uint64(max_spins), _p(status), _stream()), "zero_wait")
        return
    _check(lib().slb_zero(_p(t), c_longlong(t.numel() * t.element_size()), _stream()), "zero")


def bn_relu_pool_fwd(y, col_sum, col_sumsq, gamma, beta, running_mean, running_var, nbt, save_mean, save_invstd, out,
                     H, W, relu, pool, momentum=0.1, eps=1e-5, update_running=True, identity=False, ticket=None, flag=None,
                     seq=None, hint=None):
    P, C = y.shape[0] * y.shape[1] * y.shape[2], y.shape[3]
    _check(lib().slb_bn_relu_pool_fwd(_p(y), _p(col_sum), _p(col_sumsq), _p(gamma), _p(beta), _p(running_mean),
                                      _p(running_var), _p(nbt), _p(save_mean), _p(save_invstd), _p(out), c_int(P), c_int(C),
                                      c_int(H), c_int(W), c_int(int(relu)), c_int(int(pool)), c_float(momentum), c_float(eps),
                                      c_int(int(update_running)), c_int(int(identity)), _p(ticket), _p(flag), _p(seq), _p(hint),
                                      _dt(y), _stream()), "bn_relu_pool_fwd")


def bn_relu_pool_infer(y, gamma, beta, running_mean, running_var, out, H, W, relu, pool, eps=1e-5):
    """BatchNorm in inference mode (``invstd = rsqrt(running_var + eps)``) + ReLU + MaxPool2 on NHWC ``y``; reads the
    running statistics and writes nothing but ``out``."""
    P, C = y.shape[0] * y.shape[1] * y.shape[2], y.shape[3]
    _check(lib().slb_bn_relu_pool_infer(_p(y), _p(gamma), _p(beta), _p(running_mean), _p(running_var), _p(out), c_int(P),
                                        c_int(C), c_int(H), c_int(W), c_int(int(relu)), c_int(int(pool)), c_float(eps), _dt(y),
                                        _stream()), "bn_relu_pool_infer")


BN_BWD_CHAN_MAX_P = int(os.environ.get("SLB200_BN_BWD_CHAN_MAX_P", "4096"))


def bn_relu_pool_bwd(dout, y, gamma, beta, save_mean, save_invstd, dgamma, dbeta, dy, H, W, relu, pool, identity=False,
                     grid_bar=None, reduced=False):
    """``grid_bar`` (3+ zeroed int32 owned by the call site) selects the single-launch reduce->barrier->apply kernel.
    ``reduced``: dgamma / dbeta were already produced by ``conv3x3_dgrad(..., bn_stats=)`` -> apply pass only."""
    P, C = y.shape[0] * y.shape[1] * y.shape[2], y.shape[3]
    if reduced:
        identity, grid_bar = 2, None
    chan = (not identity) and grid_bar is None and P <= BN_BWD_CHAN_MAX_P      # one channel-owned launch (small maps)
    _check(lib().slb_bn_relu_pool_bwd(_p(dout), _p(y), _p(gamma), _p(beta), _p(save_mean), _p(save_invstd), _p(dgamma),
                                      _p(dbeta), _p(dy), c_int(P), c_int(C), c_int(H), c_int(W), c_int(int(relu)),
                                      c_int(int(pool)), c_int(int(identity)), _p(grid_bar), _dt(y), _stream()), "bn_relu_pool_bwd",
           1 if (identity or grid_bar is not None or chan) else 2)


def col_stats(y2d, col_sum, col_sumsq=None):
    P, C = y2d.shape
    _check(lib().slb_col_stats(_p(y2d), _p(col_sum), _p(col_sumsq), c_longlong(P), c_int(C), _dt(y2d), _stream()), "col_stats")


def conv3x3_small_fwd(x_nchw_f32, w_f32, bias, y, col_sum=None, col_sumsq=None):
    B, Cin, H, W = x_nchw_f32.shape
    Cout = w_f32.shape[0]
    _check(lib().slb_conv3x3_small_fwd(_p(x_nchw_f32), _p(w_f32), _p(bias), _p(y), _p(col_sum), _p(col_sumsq), c_int(B),
                                       c_int(Cin), c_int(H), c_int(W), c_int(Cout), _dt(y), _stream()), "conv3x3_small_fwd")


def conv3x3_small_wgrad(x_nchw_f32, dy, dw_f32):
    B, Cin, H, W = x_nchw_f32.shape
    Cout = dy.shape[3]
    _check(lib().slb_conv3x3_small_wgrad(_p(x_nchw_f32), _p(dy), _p(dw_f32), c_int(B), c_int(Cin), c_int(H), c_int(W),
                                         c_int(Cout), _dt(dy), _stream()), "conv3x3_small_wgrad")


def _slices(acc):
    """(parts, B, N) of a Linear result: a contiguous fp32 [parts, B, N] stack of slice partials (linear_fwd_f32 /
    linear_dgrad_f32), which the consumer adds in slice order, or a finished [B, N] buffer (parts = 0)."""
    if acc.dim() == 3:
        if acc.dtype != torch.float32 or not acc.is_contiguous():
            raise NativeError("slice partials must be a contiguous fp32 [parts, B, N] stack")
        return tuple(acc.shape)
    return (0,) + tuple(acc.shape)


def linear_finalize(acc, bias, out_bf16, out_f32, mask, relu, drop_p=0.0, seed=0, step_ptr=None):
    parts, B, N = _slices(acc)
    ldo = out_bf16.stride(0) if out_bf16 is not None else N
    _check(lib().slb_linear_finalize(_p(acc), c_int(parts), _p(bias), _p(out_bf16), _p(out_f32), _p(mask), c_int(B), c_int(N),
                                     c_int(ldo), c_int(int(relu)), c_float(drop_p), c_uint32(seed), _p(step_ptr),
                                     _dt(out_bf16) if out_bf16 is not None else c_int(0), _stream()), "linear_finalize")


def linear_bwd_prep(dacc, yout, mask, dz, dbias, relu, drop_p=0.0):
    parts, B, N = _slices(dacc)
    _check(lib().slb_linear_bwd_prep(_p(dacc), c_int(parts), _p(yout), _p(mask), _p(dz), _p(dbias), c_int(B), c_int(N),
                                     c_int(yout.stride(0) if yout is not None else N), c_int(dz.stride(0)),
                                     c_int(int(relu)), c_float(drop_p), _dt(dz), _stream()), "linear_bwd_prep")


def dropout_fwd(x, y, mask, p, seed, step_ptr=None):
    _check(lib().slb_dropout_fwd(_p(x), _p(y), _p(mask), c_longlong(x.numel()), c_float(p), c_uint32(seed), _p(step_ptr),
                                 _dt(x), _stream()), "dropout_fwd")


def dropout_bwd(dacc, mask, dx, p):
    """dx = dropout backward of dacc (mask None: a plain copy / cast; a stack of slice partials is summed first)."""
    parts = _slices(dacc)[0] if dacc.dim() == 3 else 0
    n = dacc.numel() // max(parts, 1)
    _check(lib().slb_dropout_bwd(_p(dacc), c_int(parts), _p(mask), _p(dx), c_longlong(n), c_float(p), _dt(dx), _stream()),
           "dropout_bwd")


# ---- fp32 Linear on the CUDA cores (parity mode: the reference's nn.Linear is a plain fp32 GEMM)
def linear_f32_slices(dgrad: bool, out_f: int, in_f: int) -> int:
    """Number of slice partials linear_fwd_f32 (dgrad False) or linear_dgrad_f32 (True) writes for this weight shape."""
    s = lib().slb_linear_f32_slices(c_int(int(dgrad)), c_int(out_f), c_int(in_f))
    if s < 1:
        raise NativeError(f"linear_f32_slices: bad shape {out_f}x{in_f}")
    return s


def _part_view(part, S, Bn, n):
    if part.dtype != torch.float32 or not part.is_contiguous():
        raise NativeError("partial buffer must be contiguous fp32")
    if part.numel() < S * Bn * n:
        raise NativeError(f"partial buffer too small: {part.numel()} floats < {S} slices x {Bn} x {n}")
    return part.reshape(-1)[:S * Bn * n].view(S, Bn, n)


def linear_fwd_f32(x, w, part):
    """Slice partials of x[b][in] @ w[out][in]^T in IEEE fp32 FMAs, stored into the fp32 buffer ``part`` (no zeroing
    needed).  Returns the [slices, B, out] view of ``part`` that linear_finalize (or dropout_bwd) adds up in slice order."""
    Bn, K = x.shape
    out_f = w.shape[0]
    pv = _part_view(part, linear_f32_slices(False, out_f, K), Bn, out_f)
    _check(lib().slb_linear_fwd_f32(_p(x), _p(w), _p(part), c_longlong(part.numel()), c_int(Bn), c_int(out_f), c_int(K),
                                    c_int(x.stride(0)), c_int(w.stride(0)), _stream()), "linear_fwd_f32")
    return pv


def linear_dgrad_f32(dz, w, part):
    """Slice partials of dz[b][out] @ w[out][in] into ``part``; returns the [slices, B, in] view that linear_bwd_prep or
    dropout_bwd adds up in slice order."""
    Bn = dz.shape[0]
    out_f, in_f = w.shape
    pv = _part_view(part, linear_f32_slices(True, out_f, in_f), Bn, in_f)
    _check(lib().slb_linear_dgrad_f32(_p(dz), _p(w), _p(part), c_longlong(part.numel()), c_int(Bn), c_int(out_f), c_int(in_f),
                                      c_int(dz.stride(0)), c_int(w.stride(0)), _stream()), "linear_dgrad_f32")
    return pv


def linear_wgrad_f32(dz, x, g=None, sgd=None, accumulate=False):
    """Weight gradient dz^T @ x.  ``sgd=(P, M, bias_P, bias_M, bias_G, lr, mu)``: the SGD-momentum update is applied in
    the same pass (weights and bias rows; no gradient buffer is written); otherwise ``g`` receives (or accumulates) it."""
    Bn, in_f = x.shape
    out_f = dz.shape[1]
    if sgd is not None:
        P, M, bp, bm, bg, lr, mu = sgd
        n = (Bn + 31) // 32
        _check(lib().slb_linear_wgrad_f32(_p(dz), _p(x), _p(None), _p(P), _p(M), _p(bp), _p(bm), _p(bg), c_int(Bn), c_int(out_f),
                                          c_int(in_f), c_int(dz.stride(0)), c_int(x.stride(0)), c_int(P.stride(0)), c_int(2),
                                          c_float(lr), c_float(mu), _stream()), "linear_wgrad_f32", n)
        return
    _check(lib().slb_linear_wgrad_f32(_p(dz), _p(x), _p(g), _p(None), _p(None), _p(None), _p(None), _p(None), c_int(Bn),
                                      c_int(out_f), c_int(in_f), c_int(dz.stride(0)), c_int(x.stride(0)), c_int(g.stride(0)),
                                      c_int(1 if accumulate else 0), c_float(0.0), c_float(0.0), _stream()), "linear_wgrad_f32",
           (Bn + 31) // 32)


def sumsq(g, out):
    """out[0] (zeroed by the caller) += sum(g^2) over a flat fp32 buffer."""
    _check(lib().slb_sumsq(_p(g), c_longlong(g.numel()), _p(out), _stream()), "sumsq")


def clip_scale(g, sumsq_t, max_norm: float):
    """g *= min(1, max_norm / (sqrt(sumsq) + 1e-6)) — torch.nn.utils.clip_grad_norm_ on the flat gradient."""
    _check(lib().slb_clip_scale(_p(g), c_longlong(g.numel()), _p(sumsq_t), c_float(max_norm), _stream()), "clip_scale")


def ce_fwd_bwd(logits_f32, labels_i64, dlogits_f32, loss_sum, nan_flag):
    B, C = logits_f32.shape
    _check(lib().slb_ce_fwd_bwd(_p(logits_f32), _p(labels_i64), _p(dlogits_f32), _p(loss_sum), _p(nan_flag), c_int(B),
                                c_int(C), c_int(dlogits_f32.stride(0)), _stream()), "ce_fwd_bwd")


def eval_metrics(logits_f32, labels_i64, loss_total_f64, correct_i64, count_i64):
    """Evaluation totals of one batch: loss_total += mean cross-entropy (fp64), correct += #(argmax == label) (torch.argmax
    rules: first maximum, NaN counts as the maximum), count += B.  Fixed summation order: bit-reproducible."""
    B, C = logits_f32.shape
    if logits_f32.stride(1) != 1 or logits_f32.stride(0) != C:
        raise NativeError("eval_metrics needs contiguous [B, C] logits")
    _check(lib().slb_eval_metrics(_p(logits_f32), _p(labels_i64), c_int(B), c_int(C), _p(loss_total_f64), _p(correct_i64),
                                  _p(count_i64), _stream()), "eval_metrics")


def sgd_momentum(p, g, m, p_bf16, lr, mu, first_step=False):
    _check(lib().slb_sgd_momentum(_p(p), _p(g), _p(m), _p(p_bf16), c_longlong(p.numel()), c_float(lr), c_float(mu),
                                  c_int(int(first_step)), _stream()), "sgd_momentum")


def adamw(p, g, m, v, p_bf16, lr, b1, b2, eps, wd, step, step_ptr=None):
    """``step_ptr``: device uint32 holding the step count (graph-capturable); else ``step`` is baked into the launch."""
    bc1, bc2 = 1.0 - b1 ** max(step, 1), 1.0 - b2 ** max(step, 1)
    _check(lib().slb_adamw(_p(p), _p(g), _p(m), _p(v), _p(p_bf16), c_longlong(p.numel()), c_float(lr), c_float(b1),
                           c_float(b2), c_float(eps), c_float(wd), c_float(bc1), c_float(bc2), _p(step_ptr), _stream()),
           "adamw")


def cast_f32_bf16(x, y):
    _check(lib().slb_cast_f32_bf16(_p(x), _p(y), c_longlong(x.numel()), _stream()), "cast_f32_bf16")


def fedavg(out, out_bf16, src_ptrs: Sequence[int], coefs: Sequence[float], n: int):
    k = len(src_ptrs)
    arr = (c_void_p * k)(*[c_void_p(int(s)) for s in src_ptrs])
    cf = (c_float * k)(*[float(c) for c in coefs])
    _check(lib().slb_fedavg(_p(out), _p(out_bf16), arr, cf, c_int(k), c_longlong(n), _stream()), "fedavg")


def wait_flag(flag_ptr: int, expected: int = 0, expect_ctr=None, max_spins: int = 1 << 30, status=None):
    """Stream-ordered wait until *flag >= expected (or >= *expect_ctr + 1 when a device counter is given)."""
    _check(lib().slb_wait_flag(c_void_p(flag_ptr), c_uint32(expected), _p(expect_ctr), c_uint64(max_spins), _p(status),
                               _stream()), "wait_flag")


def set_flag(flag_ptr: int, value: int = 0, seq=None, hint_ptr: int = 0):
    _check(lib().slb_set_flag(c_void_p(flag_ptr), c_uint32(value), _p(seq), c_void_p(hint_ptr), _stream()), "set_flag")


def counter_inc(ctr):
    _check(lib().slb_counter_inc(_p(ctr), _stream()), "counter_inc")


def new_stream(device, priority: int = 0):
    """A dedicated non-blocking CUDA stream wrapped for torch (``torch.cuda.ExternalStream``) — not one of torch's 32 pooled
    streams, which alias once a process has created more than 32 (see ``slb_stream_create``)."""
    out = c_void_p()
    with torch.cuda.device(device):
        _check(lib().slb_stream_create(ctypes.byref(out), c_int(1 if priority < 0 else 0)), "stream_create", 0)
    return torch.cuda.ExternalStream(out.value, device=device)


def store_u32(ptr: int, value: int):
    """Stream-ordered ``*ptr = value`` (sets the sequence counter a following graph replay publishes from)."""
    _check(lib().slb_store_u32(c_void_p(ptr), c_uint32(value), _stream()), "store_u32")


def ticket_ring_bytes(entries: int) -> int:
    return int(lib().slb_ticket_ring_bytes(c_int(entries)))


def ticket_publish(ring_ptr: int, entries: int, origin: int, it: int, gseq_ctr, batch: int):
    _check(lib().slb_ticket_publish(c_void_p(ring_ptr), c_int(entries), c_uint32(origin), c_uint32(it), _p(gseq_ctr),
                                    c_uint32(batch), _stream()), "ticket_publish")


def ticket_claim(ring_ptr: int, entries: int, total: int, max_spins: int, out_host_ptr: int):
    _check(lib().slb_ticket_claim(c_void_p(ring_ptr), c_int(entries), c_uint32(total), c_uint64(max_spins),
                                  c_void_p(out_host_ptr), _stream()), "ticket_claim")


def memcpy_async(dst_ptr: int, src_ptr: int, nbytes: int):
    _check(lib().slb_memcpy_async(c_void_p(dst_ptr), c_void_p(src_ptr), c_longlong(nbytes), _stream()), "memcpy_async", 0)


# ------------------------------------------------------------------ token-model (transformer) ops
ACT = {None: 0, "none": 0, "relu": 1, "gelu": 2, "tanh": 3}
# ``seed_ofs``: optional device uint32 mixed into the dropout seed of the token kernels.  A graph-captured training step
# passes its replay counter, so the masks baked into the graph (seeds are launch arguments) change from replay to replay.


def _gemm_bn(n: int, m: int, b_mn: bool = False) -> int:
    """Column-tile width: wide tiles unless that leaves most SMs idle."""
    m_tiles = (m + 127) // 128
    for cand in (128, 64, 32):
        if cand == 32 and b_mn:
            break
        if n >= cand and m_tiles * ((n + cand - 1) // cand) >= 96:
            return cand
    return 64 if (n > 32 or b_mn) else 32


def gemm_act(a, b, out, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldo=None, bias=None, act=None, aux=None,
             residual=None, block_n=None):
    """out_bf16[M, N] = act(A B^T + bias + residual).  A: [M, K] (K-major) or [K, M] storage (``a_mn``);
    B: [N, K] (K-major) or [K, N] storage (``b_mn``).  ``aux`` receives the pre-activation.  ``block_n`` forces the
    column-tile width (32 / 64 / 128 / 256; 32 is K-major B only); the default picks it from the shape."""
    lda = lda if lda is not None else (M if a_mn else K)
    ldb = ldb if ldb is not None else (N if b_mn else K)
    ldo = ldo if ldo is not None else N
    bn = block_n if block_n is not None else _gemm_bn(N, M, b_mn)
    _check(lib().slb_gemm_bf16_act(_p(a), _p(b), _p(out), c_int(M), c_int(N), c_int(K), c_int(int(a_mn)), c_int(int(b_mn)),
                                   c_longlong(lda), c_longlong(ldb), c_longlong(ldo), c_int(bn), _p(bias), c_int(ACT[act]),
                                   _p(aux), _p(residual), _stream()), "gemm_act")


def gemm_f32(a, b, out, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldo=None, k_split=1, block_n=None):
    """out_fp32[M, N] += A B^T (fp32 red.add epilogue: accumulates into a live gradient buffer, any ``k_split``).
    ``block_n`` as for ``gemm_act``."""
    lda = lda if lda is not None else (M if a_mn else K)
    ldb = ldb if ldb is not None else (N if b_mn else K)
    ldo = ldo if ldo is not None else N
    bn = block_n if block_n is not None else _gemm_bn(N, M, b_mn)
    _check(lib().slb_gemm_bf16(_p(a), _p(b), _p(out), c_int(M), c_int(N), c_int(K), c_int(int(a_mn)), c_int(int(b_mn)),
                               c_longlong(lda), c_longlong(ldb), c_longlong(ldo), c_int(1), c_int(max(1, k_split)), c_int(bn),
                               _stream()), "gemm_f32")


def gemm_bias_f32(a, b, out, bias, M, N, K, lda=None, ldb=None, ldo=None, block_n=None):
    """out_fp32[M, N] = A B^T + bias, plain store: A [M, K] and B [N, K] bf16, both K-major (a classifier head whose logits
    feed ``eval_metrics`` without a bf16 rounding).  ``lda`` may exceed K (rows picked out of a wider tensor)."""
    lda = lda if lda is not None else K
    ldb = ldb if ldb is not None else K
    ldo = ldo if ldo is not None else N
    bn = block_n if block_n is not None else _gemm_bn(N, M)
    _check(lib().slb_gemm_bf16_bias_f32(_p(a), _p(b), _p(out), c_int(M), c_int(N), c_int(K), c_longlong(lda), c_longlong(ldb),
                                        c_longlong(ldo), c_int(bn), _p(bias), _stream()), "gemm_bias_f32")


def patch_rows(x, out, p: int):
    """x fp32 [B, C, H, W] -> out bf16 [B * (H/p) * (W/p), C * p * p]: the unfolded patches of a Conv2d(kernel = stride = p),
    row (b, gy, gx), column (c, py, px)."""
    B, C, H, W = x.shape
    _check(lib().slb_patch_rows(_p(x), _p(out), c_int(B), c_int(C), c_int(H), c_int(W), c_int(p), _stream()), "patch_rows")


def vit_tokens(pe, cls, pos, out, B: int, P: int, E: int):
    """out bf16 [B, P+1, E] = cat(cls, pe [B, P, E]) + pos [P+1, E] (fp32 adds, one bf16 rounding)."""
    _check(lib().slb_vit_tokens(_p(pe), _p(cls), _p(pos), _p(out), c_int(B), c_int(P), c_int(E), _stream()), "vit_tokens")


def ln_rows_fwd(x, ldx: int, gamma, beta, y, rows: int, D: int, eps: float):
    """y bf16 [rows, D] = LayerNorm of the rows of ``x`` at pitch ``ldx`` elements (inference: no statistics kept)."""
    _check(lib().slb_ln_rows_fwd(_p(x), c_longlong(ldx), _p(gamma), _p(beta), _p(y), c_int(rows), c_int(D), c_float(eps),
                                 _stream()), "ln_rows_fwd")


def attn_fwd(q, k, v, ldq, ldk, ldv, q_col, k_col, v_col, out, ldo, lse, key_bias, B, S, H, Dh, p_drop=0.0, seed=0,
             seed_ofs=None):
    _check(lib().slb_attn_fwd(_p(q), _p(k), _p(v), c_longlong(ldq), c_longlong(ldk), c_longlong(ldv), c_int(q_col),
                              c_int(k_col), c_int(v_col), _p(out), c_longlong(ldo), _p(lse), _p(key_bias), c_int(B), c_int(S),
                              c_int(H), c_int(Dh), c_float(p_drop), c_uint32(seed & 0xFFFFFFFF), _p(seed_ofs), _stream()), "attn_fwd")


def attn_bwd(q, k, v, dout, ldq, ldk, ldv, lddo, q_col, k_col, v_col, do_col, dq, dk, dv, lddq, lddk, lddv, dq_col,
             dk_col, dv_col, lse, key_bias, B, S, H, Dh, p_drop=0.0, seed=0, seed_ofs=None):
    _check(lib().slb_attn_bwd(_p(q), _p(k), _p(v), _p(dout), c_longlong(ldq), c_longlong(ldk), c_longlong(ldv),
                              c_longlong(lddo), c_int(q_col), c_int(k_col), c_int(v_col), c_int(do_col), _p(dq), _p(dk),
                              _p(dv), c_longlong(lddq), c_longlong(lddk), c_longlong(lddv), c_int(dq_col), c_int(dk_col),
                              c_int(dv_col), _p(lse), _p(key_bias), c_int(B), c_int(S), c_int(H), c_int(Dh),
                              c_float(p_drop), c_uint32(seed & 0xFFFFFFFF), _p(seed_ofs), _stream()), "attn_bwd")


def ln_fwd(x, res, gamma, beta, y, pre, mean, rstd, rows, D, eps, p_drop=0.0, seed=0, seed_ofs=None):
    _check(lib().slb_ln_fwd(_p(x), _p(res), _p(gamma), _p(beta), _p(y), _p(pre), _p(mean), _p(rstd), c_int(rows), c_int(D),
                            c_float(eps), c_float(p_drop), c_uint32(seed & 0xFFFFFFFF), _p(seed_ofs), _stream()), "ln_fwd")


def ln_bwd(dy, pre, gamma, mean, rstd, dpre, dgamma, dbeta, rows, D):
    _check(lib().slb_ln_bwd(_p(dy), _p(pre), _p(gamma), _p(mean), _p(rstd), _p(dpre), _p(dgamma), _p(dbeta), c_int(rows),
                            c_int(D), _stream()), "ln_bwd")


def act_bwd(dy, ref, dz, n, kind):
    _check(lib().slb_act_bwd(_p(dy), _p(ref), _p(dz), c_longlong(n), c_int(ACT[kind]), _stream()), "act_bwd")


def colsum_bf16(x, out, rows, cols, ld=None):
    _check(lib().slb_colsum_bf16(_p(x), _p(out), c_int(rows), c_int(cols), c_longlong(ld if ld is not None else cols),
                                 _stream()), "colsum_bf16")


def dropout_bf16(x, y, n, p, seed, seed_ofs=None):
    _check(lib().slb_dropout_bf16(_p(x), _p(y), c_longlong(n), c_float(p), c_uint32(seed & 0xFFFFFFFF), _p(seed_ofs), _stream()),
           "dropout_bf16")


def embed3_fwd(ids, tts, word, pos, typ, out, tokens, S, D):
    _check(lib().slb_embed3_fwd(_p(ids), _p(tts), _p(word), _p(pos), _p(typ), _p(out), c_int(tokens), c_int(S), c_int(D),
                                _stream()), "embed3_fwd")


def embed3_bwd(ids, tts, g, dword, dpos, dtyp, tokens, S, D, pad_id=-1):
    _check(lib().slb_embed3_bwd(_p(ids), _p(tts), _p(g), _p(dword), _p(dpos), _p(dtyp), c_int(tokens), c_int(S), c_int(D),
                                c_longlong(pad_id), _stream()), "embed3_bwd")


# ------------------------------------------------------------------ GPU-resident image loader
def image_batch(data_u8, idx, dx, dy, flip, out, mean, std):
    """out[B, C, H, W] fp32 = normalise(crop/flip(data_u8[idx])); data_u8: [N, H, W, C] uint8 on the GPU,
    idx int64 [B], dx / dy / flip int32 [B] (device)."""
    B, C, H, W = out.shape
    m = (c_float * 3)(*([float(v) for v in mean] + [0.0] * (3 - len(mean))))
    sd = (c_float * 3)(*([float(v) for v in std] + [1.0] * (3 - len(std))))
    _check(lib().slb_image_batch(_p(data_u8), _p(idx), _p(dx), _p(dy), _p(flip), _p(out), c_int(B), c_int(C), c_int(H), c_int(W),
                                 m, sd, _stream()), "image_batch")


# ------------------------------------------------------------------ GPU-resident Speech Commands loader
MFCC_RECIPES = {"engine": 0, "reference": 1}          # MfccRecipe of audio.cu


def mfcc(waves, valid, out, window, fb, dct, twiddle, hop: int, preemph: float, floor: float, recipe: str = "engine"):
    """out fp32 [n, ncoef, frames] = MFCC of the fp32 waveforms [n, L] (L = win + hop * (frames - 1)), computed in fp64 with
    the fp64 tables window [win], fb [nmels, nfft/2 + 1], dct [ncoef, nmels] and twiddle [nfft, 2] (cos, sin of 2 pi j /
    nfft).  Clips whose uint8 ``valid`` byte is 0 get zero features.  ``recipe``: "engine" (fp64 pre-emphasis,
    ln(max(e, floor))) or "reference" (fp32 pre-emphasis, 20 log10(e) with e == 0 replaced by floor).  A refused call
    launches nothing."""
    if recipe not in MFCC_RECIPES:
        raise NativeError(f"mfcc: recipe must be one of {sorted(MFCC_RECIPES)}, got {recipe!r}")
    if (waves.dtype != torch.float32 or out.dtype != torch.float32 or valid.dtype != torch.uint8
            or any(t.dtype != torch.float64 for t in (window, fb, dct, twiddle))):
        raise NativeError("mfcc: waves / out fp32, valid uint8, tables fp64")
    if not all(t.is_contiguous() for t in (waves, valid, out, window, fb, dct, twiddle)):
        raise NativeError("mfcc: tensors must be contiguous")
    if waves.dim() != 2 or out.dim() != 3 or fb.dim() != 2 or dct.dim() != 2 or twiddle.dim() != 2 or twiddle.shape[1] != 2:
        raise NativeError("mfcc: waves [n, L], out [n, ncoef, frames], fb [nmels, nbins], dct [ncoef, nmels], twiddle [nfft, 2]")
    n, L = waves.shape
    ncoef, frames = out.shape[1], out.shape[2]
    nfft, nmels = twiddle.shape[0], fb.shape[0]
    if (out.shape[0] != n or valid.numel() != n or window.numel() > nfft or fb.shape[1] != nfft // 2 + 1
            or tuple(dct.shape) != (ncoef, nmels)):
        raise NativeError(f"mfcc: inconsistent shapes waves {tuple(waves.shape)} out {tuple(out.shape)} fb {tuple(fb.shape)} "
                          f"dct {tuple(dct.shape)} twiddle {tuple(twiddle.shape)}")
    _check(lib().slb_mfcc(_p(waves), _p(valid), _p(window), _p(fb), _p(dct), _p(twiddle), _p(out), c_int(n), c_int(L),
                          c_int(window.numel()), c_int(hop), c_int(frames), c_int(nfft), c_int(nmels), c_int(ncoef),
                          c_double(preemph), c_double(floor), c_int(MFCC_RECIPES[recipe]), _stream()), "mfcc")


def feature_batch(features, labels, idx, out, y):
    """out [B, ...] fp32 = features[idx], y [B] int64 = labels[idx]: one microbatch of a resident fp32 [N, ...] split
    (rows of a multiple of 4 floats, 16-byte aligned); idx int64 [B] with every entry in [0, N)."""
    if features.dtype != torch.float32 or out.dtype != torch.float32 or any(t.dtype != torch.int64 for t in (labels, idx, y)):
        raise NativeError("feature_batch: features / out fp32, labels / idx / y int64")
    if not all(t.is_contiguous() for t in (features, labels, idx, out, y)):
        raise NativeError("feature_batch: tensors must be contiguous")
    n, b = features.shape[0] if features.dim() else 0, idx.numel()
    if (labels.numel() != n or out.dim() == 0 or out.shape[0] != b or y.numel() != b
            or tuple(out.shape[1:]) != tuple(features.shape[1:])):
        raise NativeError(f"feature_batch: features {tuple(features.shape)} labels {tuple(labels.shape)} idx {tuple(idx.shape)} "
                          f"out {tuple(out.shape)} y {tuple(y.shape)}")
    d = features[0].numel() if n else 0
    _check(lib().slb_feature_batch(_p(features), _p(labels), _p(idx), _p(out), _p(y), c_int(n), c_int(b), c_longlong(d),
                                   _stream()), "feature_batch")
