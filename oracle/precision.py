"""ORACLE (test infrastructure only) - an fp64 yardstick for the fp32 sparse-convolution and dense-layer
kernels, and numpy emulators of the tensor-core operand splits.

Every layer here is a sum of products x * w.  `conv64` / `linear64` / `wgrad64` return, in fp64 over the
same terms, the reference `ref` and the magnitude `A` = the same sum with every factor replaced by its
absolute value.  The error statistic is

    e(X) = max_{j,c} |X - ref| / (A + tiny)

relative to the size of the terms, not to the size of the result, so a small output that is the sum of
large cancelling terms is held to the precision of its terms (a `|X - ref| / (1 + |ref|)` statistic lets
an output of 1e-3 be wrong by hundreds of ulps).

Acceptance criterion for the fp32-accurate modes (FFMA, 3xTF32, 3xFP16):

    e(kernel) <= KAPPA * max(e(fp32 oracle), E32_MIN)     elementwise floor (3xFP16 only) subtracted first

where the fp32 oracle is an honest fp32 computation of the same terms on the CPU
(`oracle.sparse_ops.conv_forward(..., dtype=torch.float32)`, `linear_forward`, `wgrad32`): the kernel must
be no worse than fp32 done plainly, up to KAPPA for a different summation order.  E32_MIN (one fp32 unit
roundoff) keeps the bound meaningful when the oracle happens to be exact.

3xFP16 floor (tc_common.cuh): an element more than 2^17 below its tensor's absolute maximum loses bits of
its lo part, at most 2^-39 of that maximum, so every product x * w may be off by
2^-39 (amax_x |w| + |x| amax_w) beyond the 3-pass error: `f16_floor` sums that over the terms of
each output and `err` subtracts it elementwise before dividing by A.

KAPPA = 8 was calibrated on one NVIDIA H100 80GB HBM3 at a 400 W power limit (tests/test_gpu_conv_fp64.py
prints every ratio).  Largest measured e(kernel) / max(e(fp32), E32_MIN) per kernel family, over every shape
and map of that file:

    FFMA gather-GEMM-scatter 3.7    table 3.3    ones-bits 1.0    3xTF32 6.9    3xFP16 4.0
    linear 3.0    affine 1.0    l2-normalise 1.3    weight gradient 2.1

3xTF32 is the highest: wgmma adds every k-step (8 TF32 products) into the fp32 accumulator, three passes per
k-step, and the adds do not round to nearest, so its error grows with cin / 8 * 3 adds (3xFP16 makes half as
many adds with its 16-wide k-steps).  The modes that lose bits sit far above KAPPA: 1xTF32 at 395 or more
on the same data, a 3xFP16 amax 2^20 too large at 16 or more, and the emulated 1-pass and 2-of-3-product
variants at 381 or more (tests/test_conv_precision.py requires 10 * KAPPA).
"""
import numpy as np
import torch

KAPPA = 8.0
E32_MIN = 2.0 ** -24
F16_FLOOR = 2.0 ** -39
TF32_1PASS_BOUND = 2.0 ** -10     # both operands rounded to TF32: each product within 2^-11 + 2^-11 + 2^-22
TINY = np.finfo(np.float64).tiny


def _f64(x):
  if isinstance(x, torch.Tensor):
    x = x.detach().cpu().numpy()
  return np.asarray(x, dtype=np.float64)


def _f32(x):
  if isinstance(x, torch.Tensor):
    x = x.detach().cpu().numpy()
  return np.asarray(x, dtype=np.float32)


# --------------------------------------------------------------------------- #
# fp64 references and term magnitudes
# --------------------------------------------------------------------------- #
def _conv(x, w, buckets, n_out):
  """fp64 sum over the pair lists: out[j] += x[i] @ w[kappa]."""
  x = torch.from_numpy(x)
  w = torch.from_numpy(w).reshape(len(buckets), x.shape[1], -1)
  out = torch.zeros(n_out, w.shape[2], dtype=torch.float64)
  for kap, (i, j) in enumerate(buckets):
    if len(i):
      out.index_add_(0, torch.as_tensor(j, dtype=torch.int64), x[torch.as_tensor(i, dtype=torch.int64)] @ w[kap])
  return out.numpy()


def conv64(feat, W, buckets, n_out):
  """(ref, A) fp64 [n_out, cout] of the sparse convolution out[j] = sum_{(i, j) in bucket kappa} feat[i] @ W[kappa]."""
  x, w = _f64(feat), _f64(W)
  return _conv(x, w, buckets, n_out), _conv(np.abs(x), np.abs(w), buckets, n_out)


def f16_floor(feat, W, buckets, n_out, amax_x=None, amax_w=None):
  """Absolute per-output bound [n_out, cout] of the 3xFP16 small-element loss:
  2^-39 * sum over the terms of (amax_x |w| + |x| amax_w), amax_* the tensors' true absolute maxima."""
  x, w = _f64(feat), _f64(W)
  amax_x = float(np.abs(x).max(initial=0.0)) if amax_x is None else float(amax_x)
  amax_w = float(np.abs(w).max(initial=0.0)) if amax_w is None else float(amax_w)
  return F16_FLOOR * (amax_x * _conv(np.ones_like(x), np.abs(w), buckets, n_out) +
                      amax_w * _conv(np.abs(x), np.ones_like(w), buckets, n_out))


def linear64(a, W, bias=None, b=None):
  """(ref, A) fp64 [n, cout] of concat(a, b) @ W (+ bias); W [ca + cb, cout]."""
  x = _f64(a) if b is None else np.concatenate([_f64(a), _f64(b)], 1)
  w = _f64(W).reshape(x.shape[1], -1)
  ref, A = x @ w, np.abs(x) @ np.abs(w)
  if bias is not None:
    bb = _f64(bias).reshape(1, -1)
    ref, A = ref + bb, A + np.abs(bb)
  return ref, A


def wgrad64(feat, gout, buckets):
  """(ref, A) fp64 [K, cin, cout] of the weight gradient dW[kappa] = sum_{(i, j) in bucket kappa} feat[i]^T gout[j]."""
  x, g = _f64(feat), _f64(gout)
  ref = np.zeros((len(buckets), x.shape[1], g.shape[1]))
  A = np.zeros_like(ref)
  for kap, (i, j) in enumerate(buckets):
    if len(i):
      ref[kap] = x[i].T @ g[j]
      A[kap] = np.abs(x[i]).T @ np.abs(g[j])
  return ref, A


def wgrad32(feat, gout, buckets):
  """The honest fp32 weight gradient on the CPU (torch fp32 matmul per bucket)."""
  x, g = torch.from_numpy(_f32(feat)), torch.from_numpy(_f32(gout))
  out = torch.zeros(len(buckets), x.shape[1], g.shape[1])
  for kap, (i, j) in enumerate(buckets):
    if len(i):
      out[kap] = x[torch.as_tensor(i, dtype=torch.int64)].T @ g[torch.as_tensor(j, dtype=torch.int64)]
  return out.numpy()


# --------------------------------------------------------------------------- #
# error statistic and criterion
# --------------------------------------------------------------------------- #
def err(X, ref, A, floor=None):
  """e(X) = max |X - ref| / (A + tiny), with an elementwise absolute `floor` subtracted from |X - ref| first."""
  d = np.abs(_f64(X) - ref)
  if floor is not None:
    d = np.maximum(d - floor, 0.0)
  return float((d / (A + TINY)).max(initial=0.0))


def bound(e32, kappa=KAPPA):
  """The largest e(kernel) the criterion accepts next to an fp32 oracle error e32."""
  return kappa * max(e32, E32_MIN)


def ratio(e, e32):
  """e(kernel) / max(e(fp32), E32_MIN): the quantity KAPPA bounds."""
  return e / max(e32, E32_MIN)


# --------------------------------------------------------------------------- #
# emulators of the tensor-core operand splits
# --------------------------------------------------------------------------- #
def tf32_round(x):
  """cvt.rna.tf32.f32: round to the nearest TF32 value (10 stored mantissa bits), ties away from zero."""
  u = _f32(x).view(np.uint32)
  special = (u & 0x7F800000) == 0x7F800000                   # inf / NaN pass through
  r = np.where(special, u, (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000))
  return r.astype(np.uint32).view(np.float32)


def tf32_truncate(x):
  """What the tensor core reads from an fp32 operand register: the low 13 mantissa bits dropped."""
  return (_f32(x).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32_split(x):
  """The 3xTF32 split of the kernels (split_store / pack_weight_kernel): hi = rna(x), lo = x - hi exactly in fp32.
  Returns (hi, lo) as fp32, lo as stored (the tensor core truncates it on use)."""
  x = _f32(x)
  hi = tf32_round(x)
  return hi, (x - hi).astype(np.float32)


def f16_scale_for(amax):
  """tc_common.cuh f16_scale_for: the power of two that maps amax into [2^14, 2^15); 1 for 0 / inf / NaN."""
  b = int(np.float32(amax).view(np.uint32))
  e = (b >> 23) & 255
  if e == 0 or e == 255:
    return np.float32(1.0)
  se = min(max(14 - (e - 127) + 127, 1), 254)
  return np.uint32(se << 23).view(np.float32)


def f16_split(x, amax=None):
  """The 3xFP16 split (split_store_f16 / pack_weight_f16_kernel): x' = s * x with s = f16_scale_for(amax),
  hi = fp16(x'), lo = fp16(x' - hi) (difference in fp32, both conversions round to nearest even).
  Returns (hi, lo, s) with hi / lo as fp16 arrays."""
  x = _f32(x)
  s = f16_scale_for(np.abs(x).max(initial=0.0) if amax is None else amax)
  xs = (x * s).astype(np.float32)
  hi = xs.astype(np.float16)
  lo = (xs - hi.astype(np.float32)).astype(np.float16)
  return hi, lo, s


PRODUCTS_3 = ('hh', 'lh', 'hl')     # hi*hi + lo*hi + hi*lo: the three products of the 3-pass modes


def conv_emulated(feat, W, buckets, n_out, split='tf32', products=PRODUCTS_3, amax_x=None, amax_w=None):
  """fp64 sum of the chosen split products over the pair lists: the tensor-core convolution with its
  operand rounding reproduced exactly and its accumulation made exact.  products: a subset of
  ('hh', 'lh', 'hl') (first letter: input part, second: weight part).  amax_*: the maxima the 3xFP16 scales are
  taken from (default: the true ones)."""
  if split == 'tf32':
    xh, xl = tf32_split(feat)
    wh, wl = tf32_split(W)
    xl, wl, s = tf32_truncate(xl), tf32_truncate(wl), 1.0
  elif split == 'f16':
    xh, xl, sx = f16_split(feat, amax_x)
    wh, wl, sw = f16_split(W, amax_w)
    s = float(sx) * float(sw)
  else:
    raise ValueError(split)
  parts = {'h': (xh, wh), 'l': (xl, wl)}
  out = np.zeros((n_out, np.shape(W)[-1]))
  for p in products:
    out += _conv(_f64(parts[p[0]][0]), _f64(parts[p[1]][1]), buckets, n_out)
  return out / s
