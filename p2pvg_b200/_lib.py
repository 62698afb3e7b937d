"""ctypes binding of libp2pvg_b200.so (C ABI declared in include/p2pvg_b200.h).

``CudaKernels`` is the kernel backend the engine talks to.  There is no CPU / PyTorch fallback: if the
shared library is missing the import of the product path fails loudly.
"""
from __future__ import annotations

import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libp2pvg_b200.so")

F32, BF16 = 0, 1
ACT_NONE, ACT_LRELU, ACT_TANH, ACT_SIGMOID, ACT_RELU = 0, 1, 2, 3, 4

_lib = None


class KernelError(RuntimeError):
    pass


def load_library():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(p2pvg_b200 has no CPU fallback)")
        _lib = ctypes.CDLL(LIB_PATH)
        _lib.p2pvg_last_error.restype = ctypes.c_char_p
        _lib.p2pvg_bn_workspace_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_bn_wgrad_c1_partial_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_histograms_workspace_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_png_workspace_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_png_out_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_gif_workspace_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_gif_out_bytes.restype = ctypes.c_size_t
        _lib.p2pvg_crc32c.restype = ctypes.c_uint32
        _lib.p2pvg_crc32c.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint32]
    return _lib


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"unsupported dtype {t.dtype}")


_vp = ctypes.c_void_p
_i = ctypes.c_int
_i64 = ctypes.c_int64
_f = ctypes.c_float
_d = ctypes.c_double
_sz = ctypes.c_size_t


def _p(t):
    if t is None:
        return _vp(0)
    return _vp(t.data_ptr())


class ConvFusion(ctypes.Structure):
    """p2pvg_conv_fusion_t (include/p2pvg_b200.h)."""
    _fields_ = [("fwd_stat_partial", ctypes.c_void_p), ("addend_dtype", ctypes.c_int), ("eval_scale", ctypes.c_void_p),
                ("eval_shift", ctypes.c_void_p), ("act", ctypes.c_int)]


class LstmStepModule(ctypes.Structure):
    """p2pvg_lstm_step_module (include/p2pvg_b200.h)."""
    _fields_ = [("seg_a", ctypes.c_void_p), ("idx_a", ctypes.c_void_p), ("ga", ctypes.c_int), ("seg_b", ctypes.c_void_p),
                ("idx_b", ctypes.c_void_p), ("gb", ctypes.c_int), ("tuc", ctypes.c_void_p), ("dt", ctypes.c_void_p),
                ("w_embed", ctypes.c_void_p), ("b_embed", ctypes.c_void_p), ("layers", ctypes.c_int), ("layer_w", ctypes.c_void_p),
                ("state", ctypes.c_void_p), ("head", ctypes.c_int), ("out_dim", ctypes.c_int), ("w_out", ctypes.c_void_p),
                ("b_out", ctypes.c_void_p), ("w_out2", ctypes.c_void_p), ("b_out2", ctypes.c_void_p), ("eps", ctypes.c_void_p),
                ("out", ctypes.c_void_p), ("mu", ctypes.c_void_p), ("logvar", ctypes.c_void_p), ("counter_rows", ctypes.c_int)]


LSTM_HEAD_LINEAR_TANH, LSTM_HEAD_GAUSSIAN = 0, 1


class PoseResidual(ctypes.Structure):
    """p2pvg_pose_residual (include/p2pvg_b200.h): the parameters of one residual_linear block."""
    _fields_ = [(k, ctypes.c_void_p) for k in ("w_sc", "b_sc", "w1", "b1", "w2", "b2", "w3", "b3", "gamma", "beta")]


class PoseMlpArgs(ctypes.Structure):
    """p2pvg_pose_mlp_args (include/p2pvg_b200.h)."""
    _fields_ = [("decoder", ctypes.c_int), ("g", ctypes.c_int), ("src", ctypes.c_void_p), ("src_idx", ctypes.c_void_p),
                ("fc1", PoseResidual), ("fc2", PoseResidual), ("w3", ctypes.c_void_p), ("b3", ctypes.c_void_p),
                ("skip1", ctypes.c_void_p), ("skip2", ctypes.c_void_p), ("nsrc", ctypes.c_int), ("out", ctypes.c_void_p),
                ("h1", ctypes.c_void_p), ("h2", ctypes.c_void_p)]


def pose_residual(rl):
    """PoseResidual of a models.h36m_mlp.residual_linear module (pointers to its live parameters)."""
    lins = (rl.shortcut[0], rl.long_path[0], rl.long_path[2], rl.long_path[4])
    ptrs = [t.data_ptr() for lin in lins for t in (lin.weight, lin.bias)] + [rl.norm.weight.data_ptr(), rl.norm.bias.data_ptr()]
    return PoseResidual(*ptrs)


class _Workspaces:
    """Scratch buffers of one device, shared by every CudaKernels view of it.  ``gen`` counts re-allocations: a captured
    CUDA graph that used a workspace is stale once it moved (TrainEngine.graph_generation)."""

    def __init__(self):
        self.gemm, self.bn, self.gen = {}, {}, 0


_BACKENDS = {}


def kernels_for(device):
    """The one kernel backend of a device (workspaces are allocated once per device, not per caller)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("p2pvg_b200 has no CPU path: CUDA tensors / modules only")
    idx = device.index if device.index is not None else torch.cuda.current_device()
    if idx not in _BACKENDS:
        _BACKENDS[idx] = CudaKernels(torch.device("cuda", idx))
    return _BACKENDS[idx]


class CudaKernels:
    """Launches the sm_90a kernels on the current torch CUDA stream of its device."""

    name = "cuda"

    def __init__(self, device=None):
        self.lib = load_library()
        if not torch.cuda.is_available():
            raise RuntimeError("p2pvg_b200 needs a CUDA device (no CPU fallback)")
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self._ws = _Workspaces()
        self.lane = 0   # workspace set in use: the engine switches to lane 1 for work enqueued on its side stream
        self.launches = 0
        self.gemm_flags = 0   # P2PVG_GEMM_* flags passed with every p2pvg_gemm call of this view

    def with_mode(self, tf32: bool):
        """A view of this backend (same library, same workspaces) whose fp32-operand GEMMs may (tf32=True) or may not run
        at TF32 precision.  The precision policy travels with every call; nothing is process-global."""
        import copy
        v = copy.copy(self)
        v.gemm_flags = 1 if tf32 else 0
        v.launches = 0
        return v

    @property
    def ws_gen(self):
        return self._ws.gen

    # -- helpers ---------------------------------------------------------------------------
    def _stream(self):
        return _vp(torch.cuda.current_stream(self.device).cuda_stream)

    def _ck(self, rc):
        self.launches += 1
        if rc != 0:
            raise KernelError(f"p2pvg_b200 error {rc}: {self.lib.p2pvg_last_error().decode()}")

    def gemm_workspace(self):
        ws = self._ws.gemm.get(self.lane)
        if ws is None:
            ws = self._ws.gemm[self.lane] = torch.empty(256 << 20, dtype=torch.uint8, device=self.device)
            self._ws.gen += 1
        return ws

    def bn_workspace(self, G, C):
        need = self.lib.p2pvg_bn_workspace_bytes(_i(G), _i(C))
        ws = self._ws.bn.get(self.lane)
        if ws is None or ws.numel() < need:
            ws = self._ws.bn[self.lane] = torch.empty(max(need, 16 << 20), dtype=torch.uint8, device=self.device)
            self._ws.gen += 1
        return ws

    def set_gemm_impl(self, impl: str):
        self._ck(self.lib.p2pvg_set_gemm_impl(_i({"auto": 0, "simt": 1, "tc": 2}[impl])))
        self.launches -= 1

    def set_fp32_gemm_mode(self, mode: int):
        """0: fp32 GEMMs exact on the CUDA cores; 1: K-major fp32 GEMMs on the tensor cores at TF32 precision
        (this view only; passed per call as P2PVG_GEMM_TF32)."""
        self.gemm_flags = 1 if mode else 0

    def has_tc_gemm(self) -> bool:
        return bool(self.lib.p2pvg_has_tc_gemm())

    # -- GEMM ------------------------------------------------------------------------------
    def gemm(self, A, B, C, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, ldc=None, accumulate=False, bias=None,
             addend=None, ldd=None):
        lda = lda if lda is not None else (M if a_mn else K)
        ldb = ldb if ldb is not None else (N if b_mn else K)
        ldc = ldc if ldc is not None else N
        ldd = ldd if ldd is not None else N
        assert A.dtype == B.dtype
        ws = self.gemm_workspace()
        self._ck(self.lib.p2pvg_gemm(_p(A), _i(_dt(A)), _i(int(a_mn)), _i64(lda), _p(B), _i(int(b_mn)), _i64(ldb), _p(C),
                                     _i(_dt(C)), _i64(ldc), _i(M), _i(N), _i(K), _i(int(accumulate)), _p(bias), _p(addend),
                                     _i64(ldd), _p(ws), _sz(ws.numel() if ws is not None else 0), _i(self.gemm_flags), self._stream()))

    # -- implicit-GEMM convolutions ---------------------------------------------------------
    def conv_gemm(self, kind, a, b, c, N, H, W, Ck, Cn, Cm=0, ldb=None, ldc=None, bias=None, addend=None, grp_src=None,
                  imgs_per_group=0, accumulate=False, stat_partial=None, eval_scale=None, eval_shift=None, act=ACT_NONE):
        """kind 0..5 of p2pvg_conv_gemm (see include/p2pvg_b200.h).  H, W: small-map size.  stat_partial: fp32 buffer of
        [tiles * phases, Cn, 2] receiving the BatchNorm forward statistics of the output (epilogue fusion).  eval_scale /
        eval_shift (kinds 0, 2, 3): eval-mode BatchNorm + `act` applied in the epilogue."""
        taps = 9 if kind >= 3 else 16
        if ldb is None:
            ldb = taps * Ck if kind in (0, 3, 5) else taps * Cn
        if ldc is None:
            ldc = taps * Cn if kind in (1, 4) else Cn
        ws = self.gemm_workspace()
        fusion = None
        if stat_partial is not None or eval_scale is not None or (addend is not None and addend.dtype == torch.bfloat16):
            fusion = ctypes.byref(ConvFusion(fwd_stat_partial=stat_partial.data_ptr() if stat_partial is not None else None,
                                             addend_dtype=_dt(addend) if addend is not None else F32,
                                             eval_scale=eval_scale.data_ptr() if eval_scale is not None else None,
                                             eval_shift=eval_shift.data_ptr() if eval_shift is not None else None, act=int(act)))
        self._ck(self.lib.p2pvg_conv_gemm(_i(kind), _p(a), _p(b), _i64(ldb), _p(c), _i(_dt(c)), _i64(ldc), _i(N), _i(H), _i(W), _i(Ck),
                                          _i(Cn), _i(Cm), _p(bias), _p(addend), _p(grp_src), _i(imgs_per_group), _i(int(accumulate)),
                                          _p(ws), _sz(ws.numel()), fusion, self._stream()))

    # -- conv lowering ---------------------------------------------------------------------
    def im2col(self, x, col, N, H, W, C):
        self._ck(self.lib.p2pvg_im2col_k4s2p1(_p(x), _p(col), _i(_dt(x)), _i(N), _i(H), _i(W), _i(C), self._stream()))

    def col2im(self, col, y, N, Hi, Wi, C, bias=None, col2=None, grp_src=None, imgs_per_group=0, accumulate=False):
        self._ck(self.lib.p2pvg_col2im_k4s2p1(_p(col), _p(col2), _p(grp_src), _i(imgs_per_group), _p(y), _i(_dt(col)), _i(N),
                                              _i(Hi), _i(Wi), _i(C), _p(bias), _i(int(accumulate)), self._stream()))

    def im2col3(self, x, col, N, H, W, C, ld, sgn=1):
        self._ck(self.lib.p2pvg_im2col3(_p(x), _p(col), _i(_dt(x)), _i(N), _i(H), _i(W), _i(C), _i(ld), _i(sgn), self._stream()))

    def col2im3(self, col, y, N, H, W, C, ld, bias=None):
        self._ck(self.lib.p2pvg_col2im3(_p(col), _p(y), _i(_dt(col)), _i(N), _i(H), _i(W), _i(C), _i(ld), _p(bias), self._stream()))

    def maxpool2_fwd(self, x, y, N, H, W, C):
        self._ck(self.lib.p2pvg_maxpool2_fwd(_p(x), _p(y), _i(_dt(x)), _i(N), _i(H), _i(W), _i(C), self._stream()))

    def maxpool2_bwd(self, x, dy, dx, N, H, W, C):
        self._ck(self.lib.p2pvg_maxpool2_bwd(_p(x), _p(dy), _p(dx), _i(_dt(x)), _i(N), _i(H), _i(W), _i(C), self._stream()))

    def upsample2_fwd(self, x, y, N, H, W, C):
        self._ck(self.lib.p2pvg_upsample2_fwd(_p(x), _p(y), _i(_dt(x)), _i(N), _i(H), _i(W), _i(C), self._stream()))

    def upsample2_bwd(self, dy, dx, N, H, W, C):
        self._ck(self.lib.p2pvg_upsample2_bwd(_p(dy), _p(dx), _i(_dt(dy)), _i(N), _i(H), _i(W), _i(C), self._stream()))

    def gather_add(self, dst, src, grp_src, G, n):
        self._ck(self.lib.p2pvg_gather_add(_p(dst), _i(_dt(dst)), _p(src), _p(grp_src), _i(G), _i64(n), self._stream()))

    def vgg_first_eval(self, x, nc, w, bias, scale, shift, y, N, H, W):
        """p2pvg_vgg_first_eval: fp32 NCHW frames x -> y[N,H,W,64] in y's dtype (first vgg layer, eval-mode BatchNorm)."""
        self._ck(self.lib.p2pvg_vgg_first_eval(_p(x), _i(nc), _p(w), _p(bias), _p(scale), _p(shift), _p(y), _i(_dt(y)), _i(N), _i(H),
                                               _i(W), self._stream()))

    def vgg_last_eval(self, d, w, bias, out, nc, N, H, W):
        """p2pvg_vgg_last_eval: d[N,H,W,64] -> fp32 NCHW frames out (closing ConvTranspose2d(64, nc, 3, 1, 1) + Sigmoid)."""
        self._ck(self.lib.p2pvg_vgg_last_eval(_p(d), _i(_dt(d)), _p(w), _p(bias), _p(out), _i(nc), _i(N), _i(H), _i(W), self._stream()))

    def permute4(self, src, dst, dims, strides, accumulate=False):
        d = (_i * 4)(*dims)
        s = (_i64 * 4)(*strides)
        self._ck(self.lib.p2pvg_permute4(_p(src), _i(_dt(src)), _p(dst), _i(_dt(dst)), d, s, _i(int(accumulate)), self._stream()))

    def nchw_to_nhwc_dual(self, src, dst_f32, dst_act, N, hw, C):
        """frames [N,C,hw] fp32 -> [N,hw,C] in fp32 and/or the activation dtype from one read"""
        self._ck(self.lib.p2pvg_nchw_to_nhwc_dual(_p(src), _p(dst_f32) if dst_f32 is not None else None,
                                                  _p(dst_act) if dst_act is not None else None,
                                                  _i(_dt(dst_act) if dst_act is not None else 0), _i64(N), _i(hw), _i(C), self._stream()))

    def add_indexed(self, dst, src, dst_idx, F, n):
        self._ck(self.lib.p2pvg_add_indexed(_p(dst), _p(src), _i(_dt(dst)), _p(dst_idx), _i(F), _i64(n), self._stream()))

    def transpose_batched(self, src, dst, A, P, Q):
        """dst[a][q][p] = src[a][p][q]"""
        self._ck(self.lib.p2pvg_transpose_batched(_p(src), _i(_dt(src)), _p(dst), _i(_dt(dst)), _i(A), _i(P), _i(Q), self._stream()))

    def blockdiag(self, src, dst, R, C, g):
        self._ck(self.lib.p2pvg_blockdiag(_p(src), _i(_dt(src)), _p(dst), _i(_dt(dst)), _i(R), _i(C), _i(g), self._stream()))

    def group_sum(self, inp, out, grp_src, G, F, n):
        self._ck(self.lib.p2pvg_group_sum(_p(inp), _p(out), _i(_dt(inp)), _p(grp_src), _i(G), _i(F), _i64(n), self._stream()))

    # -- batch norm ------------------------------------------------------------------------
    def bn_fwd_stats(self, x, G, R, C, gamma, beta, mean, invstd, var_unb, scale, shift, eps=1e-5):
        ws = self.bn_workspace(G, C)
        self._ck(self.lib.p2pvg_bn_fwd_stats(_p(x), _i(_dt(x)), _i(G), _i64(R), _i(C), _p(gamma), _p(beta), _f(eps), _p(ws),
                                             _sz(ws.numel()), _p(mean), _p(invstd), _p(var_unb), _p(scale), _p(shift),
                                             self._stream()))

    def bn_fwd_finalize_tiles(self, partial, parts_per_group, ldp, fold, G, R, C, gamma, beta, mean, invstd, var_unb, scale, shift, eps=1e-5):
        self._ck(self.lib.p2pvg_bn_fwd_finalize_tiles(_p(partial), _i(parts_per_group), _i(ldp), _i(fold), _i(G), _i64(R), _i(C), _p(gamma),
                                                      _p(beta), _f(eps), _p(mean), _p(invstd), _p(var_unb), _p(scale), _p(shift),
                                                      self._stream()))

    def bn_act(self, x, y, scale, shift, G, R, C, act):
        self._ck(self.lib.p2pvg_bn_act(_p(x), _p(y), _i(_dt(x)), _p(scale), _p(shift), _i(G), _i64(R), _i(C), _i(act), self._stream()))

    def bn_bwd(self, dy, x, y, mean, invstd, gamma, G, R, C, act, dx, sum_dz, sum_dzx, scale=None, shift=None):
        """y=None (LeakyReLU only): derivative recomputed from sign(x*scale+shift)."""
        ws = self.bn_workspace(G, C)
        self._ck(self.lib.p2pvg_bn_bwd(_p(dy), _p(x), _p(y), _i(_dt(x)), _p(mean), _p(invstd), _p(gamma), _i(G), _i64(R), _i(C),
                                       _i(act), _p(ws), _sz(ws.numel()), _p(dx), _p(sum_dz), _p(sum_dzx), _p(scale), _p(shift),
                                       self._stream()))

    def bn_bwd_group_sum(self, dy, x, mean, invstd, gamma, G, R, C, dx, sum_dz, sum_dzx, scale, shift, grp_src, F, dx_sum,
                         dout=None, Ho=0, wpart=None, dw=None):
        """bn_bwd (bf16, LeakyReLU from sign(x*scale+shift)) whose apply pass also writes dx_sum[f] = the sum of dx over the
        groups g with grp_src[g] == f, bit-identical to group_sum of the stored dx.  dout (C = 64): the gradient of the
        1-channel output map of the 4x4 / stride-2 ConvTranspose that reads this layer's output; its weight gradient [64][16]
        is then written to dw (wpart: bn_wgrad_c1_partial_numel(G) floats of scratch)."""
        ws = self.bn_workspace(G, C)
        wpb = wpart.numel() * wpart.element_size() if wpart is not None else 0
        self._ck(self.lib.p2pvg_bn_bwd_group_sum(_p(dy), _p(x), _p(mean), _p(invstd), _p(gamma), _i(G), _i64(R), _i(C), _p(ws),
                                                 _sz(ws.numel()), _p(dx), _p(sum_dz), _p(sum_dzx), _p(scale), _p(shift), _p(grp_src),
                                                 _i(F), _p(dx_sum), _p(dout), _i(Ho), _p(wpart), _sz(wpb), _p(dw), self._stream()))

    def bn_wgrad_c1_partial_numel(self, G):
        """fp32 elements of the per-block weight-gradient partials bn_bwd_wgrad_c1 needs for G groups."""
        return int(self.lib.p2pvg_bn_wgrad_c1_partial_bytes(_i(G))) // 4

    def bn_bwd_wgrad_c1(self, dy, x, mean, invstd, gamma, G, R, sum_dz, sum_dzx, scale, shift, cin, Ho, wpart, dw):
        """bn_bwd (bf16, LeakyReLU, C = 64) of the output of a 4x4 / stride-2 conv of the 1-channel map cin: writes that conv's
        weight gradient dw [64][16] instead of dx."""
        ws = self.bn_workspace(G, 64)
        self._ck(self.lib.p2pvg_bn_bwd_wgrad_c1(_p(dy), _p(x), _p(mean), _p(invstd), _p(gamma), _i(G), _i64(R), _p(ws), _sz(ws.numel()),
                                                _p(sum_dz), _p(sum_dzx), _p(scale), _p(shift), _p(cin), _i(Ho), _p(wpart),
                                                _sz(wpart.numel() * wpart.element_size()), _p(dw), self._stream()))

    def bn_param_grad(self, sum_dz, sum_dzx, G, C, dgamma, dbeta):
        self._ck(self.lib.p2pvg_bn_param_grad(_p(sum_dz), _p(sum_dzx), _i(G), _i(C), _p(dgamma), _p(dbeta), self._stream()))

    def bn_eval_coeffs(self, gamma, beta, rmean, rvar, C, scale, shift, eps=1e-5):
        self._ck(self.lib.p2pvg_bn_eval_coeffs(_p(gamma), _p(beta), _p(rmean), _p(rvar), _f(eps), _i(C), _p(scale), _p(shift),
                                               self._stream()))

    def bn_ema(self, rmean, rvar, mean, var_unb, order, ncalls, C, momentum=0.1):
        self._ck(self.lib.p2pvg_bn_ema(_p(rmean), _p(rvar), _p(mean), _p(var_unb), _p(order), _i(ncalls), _i(C), _f(momentum),
                                       self._stream()))

    # -- recurrent phase -------------------------------------------------------------------
    def lstm_pointwise_fwd(self, gates, c_prev, c_out, h_out, B, R):
        self._ck(self.lib.p2pvg_lstm_pointwise_fwd(_p(gates), _p(c_prev), _p(c_out), _p(h_out), _i(B), _i(R), self._stream()))

    def lstm_pointwise_bwd(self, dh, dc_next, gates, c_prev, c, dgates, dc_prev, B, R):
        self._ck(self.lib.p2pvg_lstm_pointwise_bwd(_p(dh), _p(dc_next), _p(gates), _p(c_prev), _p(c), _p(dgates), _p(dc_prev), _i(B),
                                                   _i(R), self._stream()))

    def lstm_scan_fwd(self, pre, whh, bhh, gates, hs, cs, S, B, R, counter, tf32=False):
        self._ck(self.lib.p2pvg_lstm_scan_fwd(_p(pre), _p(whh), _p(bhh), _p(gates), _p(hs), _p(cs), _i(S), _i(B), _i(R), _i(int(tf32)),
                                              _p(counter), self._stream()))

    def lstm_scan_bwd(self, dhtop, whh, gates, cs, dG, S, B, R, counter, tf32=False):
        self._ck(self.lib.p2pvg_lstm_scan_bwd(_p(dhtop), _p(whh), _p(gates), _p(cs), _p(dG), _i(S), _i(B), _i(R), _i(int(tf32)),
                                              _p(counter), self._stream()))

    def lstm_step(self, modules, rows, R):
        """p2pvg_lstm_step: modules = list of one or two dicts of LstmStepModule fields (tensors or None; ints as ints)."""
        arr = (LstmStepModule * len(modules))()
        for i, m in enumerate(modules):
            for k, v in m.items():
                setattr(arr[i], k, v if isinstance(v, int) else (v.data_ptr() if v is not None else None))
        self._ck(self.lib.p2pvg_lstm_step(arr, _i(len(modules)), _i(rows), _i(R), self._stream()))

    def pose_mlp(self, mod, decoder, src, out, rows, src_idx=None, skips=None, nsrc=0, h1=None, h2=None):
        """p2pvg_pose_mlp: one call of a models.h36m_mlp encoder (decoder=False; h1 / h2 receive the skips when given) or
        decoder (decoder=True; skips = [h1, h2] of an encoder call on nsrc rows) on `rows` rows of src[src_idx[0]]."""
        s1, s2 = skips if skips is not None else (None, None)
        a = PoseMlpArgs(decoder=int(decoder), g=mod.fc1.norm.normalized_shape[0], src=src.data_ptr(),
                        src_idx=src_idx.data_ptr() if src_idx is not None else None, fc1=pose_residual(mod.fc1),
                        fc2=pose_residual(mod.fc2), w3=mod.fc3.weight.data_ptr(), b3=mod.fc3.bias.data_ptr(),
                        skip1=s1.data_ptr() if s1 is not None else None, skip2=s2.data_ptr() if s2 is not None else None,
                        nsrc=int(nsrc), out=out.data_ptr(), h1=h1.data_ptr() if h1 is not None else None,
                        h2=h2.data_ptr() if h2 is not None else None)
        self._ck(self.lib.p2pvg_pose_mlp(ctypes.byref(a), _i(rows), self._stream()))

    def reparam_kl_fwd(self, mu, lv, mu_p, lv_p, eps, eps_p, z, z_p, n, kl_sum):
        self._ck(self.lib.p2pvg_reparam_kl_fwd(_p(mu), _p(lv), _p(mu_p), _p(lv_p), _p(eps), _p(eps_p), _p(z), _p(z_p), _i(n),
                                               _p(kl_sum), self._stream()))

    def reparam_kl_bwd(self, mu, lv, mu_p, lv_p, eps, eps_p, dz, dz_p, kl_coef, dmu, dlv, dmu_p, dlv_p, n):
        self._ck(self.lib.p2pvg_reparam_kl_bwd(_p(mu), _p(lv), _p(mu_p), _p(lv_p), _p(eps), _p(eps_p), _p(dz), _p(dz_p),
                                               _f(kl_coef), _p(dmu), _p(dlv), _p(dmu_p), _p(dlv_p), _i(n), self._stream()))

    def build_concat(self, dst, A, ia, ga, Bm, ib, gb, tuc, dt, S, B, ld=None):
        self._ck(self.lib.p2pvg_build_concat(_p(dst), _p(A), _p(ia), _i(ga), _p(Bm), _p(ib), _i(gb), _p(tuc), _p(dt), _i(S), _i(B),
                                             _i(ld if ld is not None else ga + gb + 2), self._stream()))

    def gather_add_cols(self, dst, src, idx, S, T, B, g, W, col0, init=False):
        self._ck(self.lib.p2pvg_gather_add_cols(_p(dst), _p(src), _p(idx), _i(S), _i(T), _i(B), _i(g), _i(W), _i(col0),
                                                _i(int(init)), self._stream()))

    def align(self, H, in_idx, h_pred, P, B, g, coef, loss_partial, d_hpred, dH):
        self._ck(self.lib.p2pvg_align(_p(H), _p(in_idx), _p(h_pred), _i(P), _i(B), _i(g), _f(coef), _p(loss_partial), _p(d_hpred),
                                      _p(dH), self._stream()))

    def colsum(self, x, rows, cols, ld, out, accumulate=False):
        ws = self.bn_workspace(1, 1)
        self._ck(self.lib.p2pvg_colsum(_p(x), _i(_dt(x)), _i64(rows), _i(cols), _i64(ld), _p(out), _i(int(accumulate)), _p(ws),
                                       _sz(ws.numel()), self._stream()))

    def act_fwd(self, x, n, act):
        self._ck(self.lib.p2pvg_act_fwd(_p(x), _i64(n), _i(act), self._stream()))

    def act_bwd(self, dy, y, dx, n, act):
        self._ck(self.lib.p2pvg_act_bwd(_p(dy), _p(y), _p(dx), _i64(n), _i(act), self._stream()))

    # -- losses / optimiser ----------------------------------------------------------------
    def mse_chunks(self):
        return int(self.lib.p2pvg_mse_chunks())

    def sigmoid_mse(self, raw, x, tgt, coef, G, E, pred, d_raw, partial):
        self._ck(self.lib.p2pvg_sigmoid_mse(_p(raw), _i(_dt(raw)), _p(x), _p(tgt), _p(coef), _i(G), _i64(E), _p(pred), _p(d_raw),
                                            _p(partial), self._stream()))

    def convt_c1_loss(self, col, col2, grp_src, bias, x, tgt, coef, G, B, Hi, Wi, d_raw, partial, C=1):
        self._ck(self.lib.p2pvg_convt_c1_loss(_p(col), _p(col2), _i(_dt(col)), _p(grp_src), _p(bias), _p(x), _p(tgt), _p(coef), _i(G), _i(B),
                                              _i(Hi), _i(Wi), _i(C), _p(d_raw), _p(partial), self._stream()))

    def layernorm_fwd(self, x, gamma, beta, y, mean, rstd, rows, C, eps=1e-5):
        self._ck(self.lib.p2pvg_layernorm_fwd(_p(x), _p(gamma), _p(beta), _p(y), _p(mean), _p(rstd), _i64(rows), _i(C), _f(eps), self._stream()))

    def layernorm_bwd(self, dy, x, mean, rstd, gamma, dx, dgamma, dbeta, rows, C):
        ws = self.bn_workspace(1, 1)
        self._ck(self.lib.p2pvg_layernorm_bwd(_p(dy), _p(x), _p(mean), _p(rstd), _p(gamma), _p(dx), _p(dgamma), _p(dbeta), _i64(rows), _i(C),
                                              _p(ws), _sz(ws.numel()), self._stream()))

    def mse_plain(self, pred, x, tgt, coef, G, E, d_pred, partial):
        self._ck(self.lib.p2pvg_mse_plain(_p(pred), _p(x), _p(tgt), _p(coef), _i(G), _i64(E), _p(d_pred), _p(partial), self._stream()))

    def publish_scalars(self, src, n, host_pinned, seq):
        """src[0..n) + *seq -> page-locked host memory (zero-copy store from the device)"""
        self._ck(self.lib.p2pvg_publish_scalars(_p(src), _i(n), _vp(host_pinned.data_ptr()), _p(seq), self._stream()))

    def finalize_losses(self, mse_partial, n_recon, has_cpc, E, kl_sum, batch_size, align_partial, n_align, seq_len, out):
        self._ck(self.lib.p2pvg_finalize_losses(_p(mse_partial), _i(n_recon), _i(int(has_cpc)), _d(float(E)), _p(kl_sum),
                                                _f(batch_size), _p(align_partial), _i(n_align), _f(seq_len), _p(out),
                                                self._stream()))

    def seq_losses(self, rec, sigmoid, x, tgt, S, B, E, mu, lv, mu_p, lv_p, z, H, in_idx, h_pred, g, has_cpc, batch_size, seq_len,
                   partial, counter, per_seq, out):
        """p2pvg_seq_losses: per_seq fp64 [4, B] (mse, kld, cpc, align of every row) and out fp64 [4] of an eval-mode forward;
        partial fp64 [(S + 1) * B * 3] and counter int32 [1] (zero before the first launch, left zero) are its workspace."""
        assert partial.dtype == per_seq.dtype == out.dtype == torch.float64 and counter.dtype == torch.int32
        self._ck(self.lib.p2pvg_seq_losses(_p(rec), _i(_dt(rec)), _i(int(sigmoid)), _p(x), _p(tgt), _i(S), _i(B), _i64(E), _p(mu), _p(lv),
                                           _p(mu_p), _p(lv_p), _i(z), _p(H), _p(in_idx), _p(h_pred), _i(g), _i(int(has_cpc)),
                                           _d(float(batch_size)), _d(float(seq_len)), _p(partial), _p(counter), _p(per_seq), _p(out),
                                           self._stream()))

    def adam(self, p, g, m, v, n, lr, beta1, beta2, eps, step_t):
        self._ck(self.lib.p2pvg_adam_legacy(_p(p), _p(g), _p(m), _p(v), _i64(n), _d(lr), _d(beta1), _d(beta2), _d(eps),
                                            _p(step_t), self._stream()))

    def scale(self, x, n, a):
        self._ck(self.lib.p2pvg_scale(_p(x), _i64(n), _f(a), self._stream()))

    # -- data ------------------------------------------------------------------------------
    def moving_mnist(self, digits, draws, out, T, B, S, num_digits, deterministic):
        """digits uint8 [N,32,32], draws int32 [B,num_digits,stride], out fp32 [T,B,1,S,S] (p2pvg_moving_mnist)."""
        assert digits.dtype == torch.uint8 and draws.dtype == torch.int32 and out.dtype == torch.float32
        assert digits.is_contiguous() and draws.is_contiguous() and out.is_contiguous()
        self._ck(self.lib.p2pvg_moving_mnist(_p(digits), _i(digits.shape[0]), _p(draws), _i(draws.shape[-1]), _p(out), _i(T), _i(B),
                                             _i(S), _i(num_digits), _i(int(deterministic)), self._stream()))

    def video_windows(self, frames, clip_first, clip_len, entries, draws, paired_flips, L, out):
        """frames uint8 [F,C,H,W], clip_first int64 / clip_len int32 [n_clips], entries int32 [B], draws int32 [B] or None,
        out fp32 [T,B,C,H,W] (p2pvg_video_windows)."""
        assert frames.dtype == torch.uint8 and clip_first.dtype == torch.int64 and clip_len.dtype == torch.int32
        assert entries.dtype == torch.int32 and (draws is None or draws.dtype == torch.int32) and out.dtype == torch.float32
        assert all(t is None or t.is_contiguous() for t in (frames, clip_first, clip_len, entries, draws, out))
        T, B, C, H, W = out.shape
        assert frames.dim() == 4 and tuple(frames.shape[1:]) == (C, H, W) and len(entries) == B
        assert len(clip_len) == len(clip_first) and (draws is None or len(draws) == B)
        self._ck(self.lib.p2pvg_video_windows(_p(frames), _p(clip_first), _p(clip_len), _i(len(clip_len)), _p(entries), _p(draws),
                                              _i(int(paired_flips)), _i(B), _i(L), _i(T), _i(C), _i(H), _i(W), _p(out),
                                              self._stream()))

    def pose_windows(self, pose_2d, pose_3d, seq_first, seq_len, entries, draws, speed_range, L, out_2d, out_3d):
        """pose_2d fp32 [F,J,2], pose_3d fp32 [F,J,3], seq_first int64 / seq_len int32 [n_seq], entries int32 [B], draws int32
        [2,B], out_2d fp32 [T,B,J,2], out_3d fp32 [T,B,J,3] (p2pvg_pose_windows)."""
        assert pose_2d.dtype == pose_3d.dtype == out_2d.dtype == out_3d.dtype == torch.float32
        assert seq_first.dtype == torch.int64 and seq_len.dtype == entries.dtype == draws.dtype == torch.int32
        assert all(t.is_contiguous() for t in (pose_2d, pose_3d, seq_first, seq_len, entries, draws, out_2d, out_3d))
        T, B, J, _ = out_2d.shape
        F = pose_2d.shape[0]
        assert tuple(pose_2d.shape) == (F, J, 2) and tuple(pose_3d.shape) == (F, J, 3) and tuple(out_3d.shape) == (T, B, J, 3)
        assert len(seq_len) == len(seq_first) and len(entries) == B and tuple(draws.shape) == (2, B)
        self._ck(self.lib.p2pvg_pose_windows(_p(pose_2d), _p(pose_3d), _i(J), _p(seq_first), _p(seq_len), _i(len(seq_len)),
                                             _p(entries), _p(draws), _i(B), _i(speed_range[0]), _i(speed_range[1]), _i(L), _i(T),
                                             _p(out_2d), _p(out_3d), self._stream()))

    # -- metrics ---------------------------------------------------------------------------
    def frame_metrics(self, pred, gt, pairs, n_pairs, C, H, W, data_range, out):
        """p2pvg_frame_metrics: out fp64 [n_pairs, 3] = mse, psnr, ssim of pred[pairs[p, 0]] against gt[pairs[p, 1]]
        (fp32 [.., C, H, W] stores, int32 pairs; checked by p2pvg_b200.metrics)."""
        self._ck(self.lib.p2pvg_frame_metrics(_p(pred), _p(gt), _p(pairs), _i(n_pairs), _i(C), _i(H), _i(W), _f(data_range), _p(out),
                                              self._stream()))

    def pose_metrics(self, pred, gt, pairs, n_pairs, J, out):
        """p2pvg_pose_metrics: out fp64 [n_pairs, 2] = mse, mpjpe of pred[pairs[p, 0]] against gt[pairs[p, 1]] ([.., J, 3])."""
        self._ck(self.lib.p2pvg_pose_metrics(_p(pred), _p(gt), _p(pairs), _i(n_pairs), _i(J), _p(out), self._stream()))

    def metrics_fold(self, scores, higher_mask, B, nsample, segs, col_bin, part_v, part_c, counter, sums, counts, rows):
        """p2pvg_metrics_fold: scores fp64 [n_pairs, n_metrics] folded into the bins sums fp64 [n_bins, n_metrics, 3], counts
        int64 [n_bins, n_metrics, 4] and rows int64 [n_bins]; segs int32 [n_seg, 3] and col_bin int32 [n_cols] device tables
        (checked by p2pvg_b200.evaluate); part_v fp64 / part_c int32 [n_cols * B * n_metrics * 2] and counter int32 [1]
        (zero before the first launch, left zero) are its workspace."""
        nm = scores.shape[1]
        assert scores.dtype == sums.dtype == part_v.dtype == torch.float64 and counts.dtype == rows.dtype == torch.int64
        assert segs.dtype == col_bin.dtype == part_c.dtype == counter.dtype == torch.int32
        assert part_v.numel() >= col_bin.numel() * B * nm * 2 and part_c.numel() >= col_bin.numel() * B * nm * 2
        assert tuple(sums.shape[1:]) == (nm, 3) and tuple(counts.shape) == (sums.shape[0], nm, 4) and rows.numel() == sums.shape[0]
        self._ck(self.lib.p2pvg_metrics_fold(_p(scores), _i(nm), _i(higher_mask), _i(B), _i(nsample), _p(segs), _i(segs.shape[0]),
                                             _p(col_bin), _i(col_bin.numel()), _i(sums.shape[0]), _p(part_v), _p(part_c),
                                             _p(counter), _p(sums), _p(counts), _p(rows), self._stream()))

    # -- qualitative pictures ----------------------------------------------------------------
    def vis_canvas(self, store0, n0, store1, n1, C, H, tiles_host, tiles_dev, r_len, n_block, canvas, video, gif):
        """p2pvg_vis_canvas: the PNG canvas, video tensor and GIF frames of misc/visualize.py vis_seq from fp32 frame stores
        [n, C, H, H] and the int32 tile table [r_len, n_block, 6, 3] (tiles_host on the host, tiles_dev its device copy;
        checked by the library before the launch)."""
        self._ck(self.lib.p2pvg_vis_canvas(_p(store0), _i(n0), _p(store1), _i(n1), _i(C), _i(H), _vp(tiles_host.ctypes.data),
                                           _p(tiles_dev), _i(r_len), _i(n_block), _p(canvas), _p(video), _p(gif), self._stream()))

    def vis_tiles(self, store0, n0, store1, n1, C, H, tiles_host, images_host, tables_dev, out_f, out_u8):
        """p2pvg_vis_tiles: the tiles of the int32 host table tiles_host [n, 6] (store, frame, border, image, y, x) written into
        the destination images of the int64 host table images_host [m, 4] (offset, kind, h, w) in out_f (fp32) / out_u8
        (uint8); tables_dev: a device workspace of 32 m + 24 n bytes.  Checked by the library before the launch."""
        self._ck(self.lib.p2pvg_vis_tiles(_p(store0), _i(n0), _p(store1), _i(n1), _i(C), _i(H), _vp(tiles_host.ctypes.data),
                                          _i(len(tiles_host)), _vp(images_host.ctypes.data), _i(len(images_host)), _p(tables_dev),
                                          _p(out_f), ctypes.c_longlong(0 if out_f is None else out_f.numel()), _p(out_u8),
                                          ctypes.c_longlong(0 if out_u8 is None else out_u8.numel()), self._stream()))

    # -- TensorBoard histograms ------------------------------------------------------------
    def histograms_workspace_bytes(self, segs_host, n_edges):
        """Bytes of workspace p2pvg_histograms needs for the int64 host segment table segs_host [n_seg, 3]."""
        return int(self.lib.p2pvg_histograms_workspace_bytes(_vp(segs_host.ctypes.data), _i(len(segs_host)), _i(n_edges)))

    def histograms(self, segs_host, edges_host, workspace, counts, stats):
        """p2pvg_histograms: counts int64 [n_seg, n_edges - 1] and stats fp64 [n_seg, 5] (min, max, num, sum, sum_squares) of
        the segments of segs_host (int64 [n_seg, 3] on the host: address, count, P2PVG_F32 / P2PVG_F64) over the fp64 host
        edge table edges_host (both checked by the library before the launch)."""
        self._ck(self.lib.p2pvg_histograms(_vp(segs_host.ctypes.data), _i(len(segs_host)), _vp(edges_host.ctypes.data),
                                           _i(len(edges_host)), _p(workspace), _sz(workspace.numel() * workspace.element_size()),
                                           _p(counts), _p(stats), self._stream()))

    # -- PNG files -----------------------------------------------------------------------------
    def png_bytes(self, images_host):
        """(workspace bytes, output bytes) p2pvg_png_encode needs for the int64 host image table images_host [n, 5]
        (address, dtype, C, H, W); (0, 0) for a table it rejects."""
        ptr, n = _vp(images_host.ctypes.data), _i(len(images_host))
        return int(self.lib.p2pvg_png_workspace_bytes(ptr, n)), int(self.lib.p2pvg_png_out_bytes(ptr, n))

    def png_encode(self, images_host, rule, workspace, out, files):
        """p2pvg_png_encode: the PNG files of the images of images_host (checked by the library before any launch) packed into
        the uint8 device buffer out, with their (offset, size) in the int64 device tensor files [n, 2]."""
        self._ck(self.lib.p2pvg_png_encode(_vp(images_host.ctypes.data), _i(len(images_host)), _i(rule), _p(workspace),
                                           _sz(workspace.numel()), _p(out), _sz(out.numel()), _p(files), self._stream()))

    # -- GIF files -----------------------------------------------------------------------------
    def gif_bytes(self, anims_host):
        """(workspace bytes, output bytes) p2pvg_gif_encode needs for the int64 host animation table anims_host [n, 7]
        (address, dtype, T, H, W, delay, loop); (0, 0) for a table it rejects."""
        ptr, n = _vp(anims_host.ctypes.data), _i(len(anims_host))
        return int(self.lib.p2pvg_gif_workspace_bytes(ptr, n)), int(self.lib.p2pvg_gif_out_bytes(ptr, n))

    def gif_encode(self, anims_host, rule, workspace, out, files):
        """p2pvg_gif_encode: the GIF files of the animations of anims_host (checked by the library before any launch) packed
        into the uint8 device buffer out, with their (offset, size) in the int64 device tensor files [n, 2]."""
        self._ck(self.lib.p2pvg_gif_encode(_vp(anims_host.ctypes.data), _i(len(anims_host)), _i(rule), _p(workspace),
                                           _sz(workspace.numel()), _p(out), _sz(out.numel()), _p(files), self._stream()))


def crc32c(data, crc=0):
    """p2pvg_crc32c: the CRC-32C of the bytes ``data``, continuing from ``crc``.  Host code: needs the library, no device."""
    data = bytes(data)
    return int(load_library().p2pvg_crc32c(data, len(data), crc))
