"""The packed weight formats and activation layouts the kernels read, each written down once (DESIGN.md §3).

Activations are NHWC rows ``[(n, y, x), C]`` in the activation dtype (bf16, or fp32 in parity mode); frames come in and
go out as NCHW fp32.  Convolution weights are kept as fp32 masters in PyTorch's layout and packed into GEMM operands in
the activation dtype (tap = kh * k + kw):

  conv 4x4          W[Cout, Cin, 4, 4]  -> [Cout][tap][Cin]     also the final 4x4-valid conv of the encoders
  ConvTranspose 4x4 W[Cin, Cout, 4, 4]  -> [Cin][tap][Cout]     also upc1, the 1x1 -> 4x4 ConvTranspose of the decoders
  conv 3x3          W[Cout, Cin, 3, 3]  -> [Cout][tap][Cin]     rows padded to up8(9 Cin)
  conv 3x3, data gradient               -> [Cin][tap][Cout]

Each unpack_* is the inverse of its pack: it turns an fp32 weight gradient computed in the packed layout into PyTorch's
layout.  ``K`` is the kernel backend (``_lib.CudaKernels``, or any object with the same methods).
"""


def up8(n):
    """n rounded up to a multiple of 8: a row of that many bf16 or fp32 elements is a multiple of 16 bytes (TMA pitch)."""
    return (n + 7) // 8 * 8


def implicit_shape(cin, cout):
    """Whether the implicit-GEMM convolution kernels (p2pvg_conv_gemm) take a layer with these channel counts."""
    return cin % 64 == 0 and cout % 64 == 0


# ---- 4x4 convolutions ---------------------------------------------------------------------------------------------
def pack_conv4(K, w, out):
    """Conv W[Cout, Cin, 4, 4] -> out[Cout][tap][Cin]."""
    K.transpose_batched(w, out, w.shape[0], w.shape[1], 16)


def pack_convt4(K, w, out):
    """ConvTranspose W[Cin, Cout, 4, 4] -> out[Cin][tap][Cout]."""
    K.transpose_batched(w, out, w.shape[0], w.shape[1], 16)


def unpack_conv4(K, gw, out):
    """gw[Cout][tap][Cin] -> out[Cout, Cin, 4, 4] (inverse of pack_conv4)."""
    K.transpose_batched(gw, out, out.shape[0], 16, out.shape[1])


def unpack_convt4(K, gw, out):
    """gw[Cin][tap][Cout] -> out[Cin, Cout, 4, 4] (inverse of pack_convt4)."""
    K.transpose_batched(gw, out, out.shape[0], 16, out.shape[1])


def tile_bias(K, b, out, reps):
    """out[reps][C] = b[C] for every rep: the bias of a GEMM whose output row holds reps taps or pixels of C channels."""
    K.permute4(b, out, (reps, b.numel(), 1, 1), (0, 1, 0, 0))


# ---- 3x3 convolutions ---------------------------------------------------------------------------------------------
def pack_conv3(K, w, out, c0=0, cin=None, scratch=None):
    """Conv W[Cout, Cin_total, 3, 3], input channels [c0, c0 + cin) (default: all) -> out[Cout][tap][cin] with the row
    pitch padded to up8(9 cin).  When 9 cin is not a multiple of 8 the rows are first packed unpadded into scratch
    (Cout * 9 cin + 8 elements) and re-pitched from there: the pad columns pick up the next row's first weights, or the
    8 slack elements after the last row, all finite, and only ever meet zero columns of the other operand."""
    cout, cin_total = w.shape[0], w.shape[1]
    cin = cin or cin_total
    ld = up8(9 * cin)
    dense = out if ld == 9 * cin else scratch
    K.permute4(w.view(-1)[c0 * 9:], dense, (cout, 3, 3, cin), (cin_total * 9, 3, 1, 9))
    if dense is not out:
        K.permute4(dense, out, (cout, ld, 1, 1), (9 * cin, 1, 0, 0))


def pack_conv3_t(K, w, out, c0=0, cin=None):
    """Conv W[Cout, Cin_total, 3, 3], input channels [c0, c0 + cin) (default: all) -> out[cin][tap][Cout], the weight
    operand of the data gradient."""
    cout, cin_total = w.shape[0], w.shape[1]
    cin = cin or cin_total
    K.permute4(w.view(-1)[c0 * 9:], out, (cin, 3, 3, cout), (9, 3, 1, cin_total * 9))


def unpack_conv3(K, gw, out, halves=1):
    """gw[halves][Cout][tap][Cin] with the row pitch up8(9 Cin) -> out[Cout, halves * Cin, 3, 3] (inverse of pack_conv3).
    halves = 2: the two input-channel halves of a torch.cat input, packed separately with c0 = 0 and c0 = Cin."""
    cout, cin = out.shape[0], out.shape[1] // halves
    ld = up8(9 * cin)
    K.permute4(gw, out, (cout, halves, cin, 9), (ld, cout * ld, 1, cin))


# ---- activations --------------------------------------------------------------------------------------------------
def nchw_to_nhwc(K, x, out, N, hw, C):
    """Frames x[N, C, hw] -> out[N, hw, C] in out's dtype."""
    K.permute4(x, out, (N, hw, C, 1), (C * hw, 1, hw, 0))


def nhwc_to_nchw(K, a, out, N, hw, C):
    """Rows a[N, hw, C] -> out[N, C, hw] in out's dtype."""
    K.permute4(a, out, (N, C, hw, 1), (hw * C, 1, C, 0))


def cast(K, src, out, n):
    """out[:n] = src[:n] in out's dtype (a plain copy when the dtypes match)."""
    K.permute4(src, out, (n, 1, 1, 1), (1, 0, 0, 0))
