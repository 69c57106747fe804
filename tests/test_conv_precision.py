"""The fp64 yardstick of oracle/precision.py on the CPU: its emulators follow the kernels' rounding rules, and its
criterion tells the accurate tensor-core modes from the lossy ones before any GPU run.

On realistic kernel maps the emulated 3xTF32 and 3xFP16 convolutions (operand splits reproduced exactly, sums
exact) meet e <= KAPPA * e(fp32 oracle); the emulated 1-pass modes and every variant that drops one of the three
products miss it by at least 10x."""
import numpy as np
import pytest
import torch

from oracle import precision as pr
from oracle import sparse_ops as so


def _coords(seed, n, D, span):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-span, span, size=(n, D)), axis=0)
  c = c[g.permutation(len(c))]
  return np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)


def _tf32_rna_reference(x):
  """Round to 11 significant bits, ties away from zero, in fp64 arithmetic (independent of the bit trick)."""
  x = np.asarray(x, np.float64)
  m, e = np.frexp(x)                                   # x = m 2^e, 0.5 <= |m| < 1
  return (np.sign(m) * np.floor(np.abs(m) * 2.0 ** 11 + 0.5) * 2.0 ** (e - 11)).astype(np.float32)


def test_tf32_round_is_round_to_nearest_ties_away():
  ties = np.array([1 + 2 ** -11, -(1 + 2 ** -11), 1 + 5 * 2 ** -11, -(1 + 5 * 2 ** -11)], np.float32)
  assert pr.tf32_round(ties).tolist() == [1 + 2 ** -10, -(1 + 2 ** -10), 1 + 3 * 2 ** -10, -(1 + 3 * 2 ** -10)]
  g = np.random.default_rng(0)
  x = (g.standard_normal(200000) * np.exp(g.uniform(-40, 40, 200000))).astype(np.float32)
  x[:4] = [0.0, -0.0, 1.0, -3.0]
  hi, lo = pr.tf32_split(x)
  assert np.array_equal(hi, _tf32_rna_reference(x))
  assert not (hi.view(np.uint32) & 0x1FFF).any()                  # 10 stored mantissa bits
  # the identity the packed weights satisfy (hi tile + lo tile == W, exactly, in fp32)
  assert np.array_equal(hi + lo, x)
  assert (np.abs(lo) <= 2.0 ** -11 * np.abs(x)).all()
  assert np.array_equal(pr.tf32_truncate(np.float32(1 + 2 ** -11 + 2 ** -20)), np.float32(1.0))


def test_f16_split_and_scale():
  for amax in (1e-30, 3e-5, 1.0, 4.0, 7.9, 6e4, 3e38):
    s = float(pr.f16_scale_for(amax))
    assert 2.0 ** 14 <= amax * s < 2.0 ** 15 and np.log2(s) == round(np.log2(s)), (amax, s)
  assert pr.f16_scale_for(0.0) == 1.0 and pr.f16_scale_for(np.inf) == 1.0
  g = np.random.default_rng(1)
  x = (g.standard_normal(100000) * np.exp(g.uniform(-20, 0, 100000))).astype(np.float32)
  x[0] = 2.5
  hi, lo, s = pr.f16_split(x)
  rec = (hi.astype(np.float64) + lo.astype(np.float64)) / float(s)
  big = np.abs(x) >= 2.0 ** -17 * 2.5
  # 2^-22 relative above the threshold; below it lo loses bits, at most 2^-39 of the maximum
  assert (np.abs(rec - x)[big] <= 2.0 ** -22 * np.abs(x[big])).all()
  assert (np.abs(rec - x) <= 2.0 ** -22 * np.abs(x) + 2.0 ** -39 * 2.5).all()
  assert (~big).sum() > 100


def test_references_and_magnitudes():
  c = _coords(3, 1500, 3, 8)
  n = len(c)
  b = so.kernel_map(c, c, so.kernel_offsets(3, 3, 1))
  g = torch.Generator().manual_seed(0)
  x, W = torch.randn(n, 8, generator=g), torch.randn(27, 8, 5, generator=g)
  ref, A = pr.conv64(x, W, b, n)
  assert np.allclose(ref, so.conv_forward(x, W, b, n, dtype=torch.float64).numpy(), rtol=0, atol=1e-12)
  assert (A >= np.abs(ref)).all()
  gout = torch.randn(n, 5, generator=g)
  dref, dA = pr.wgrad64(x, gout, b)
  # the weight gradient is the adjoint of the convolution: <conv(x, W), gout> == <W, dW>
  assert np.isclose((ref * gout.double().numpy()).sum(), (W.double().numpy() * dref).sum(), rtol=1e-12)
  assert (dA >= np.abs(dref)).all()
  a, bb, Wl, bias = x[:, :5], x[:, 5:], torch.randn(8, 3, generator=g), torch.randn(3, generator=g)
  lref, lA = pr.linear64(a, Wl, bias, bb)
  assert np.allclose(lref, (x.double() @ Wl.double() + bias.double()).numpy(), rtol=0, atol=1e-12)
  assert (lA >= np.abs(lref)).all()


VARIANTS = {'1xTF32': ('tf32', ('hh',)), 'TF32 hh+lh': ('tf32', ('hh', 'lh')), 'TF32 hh+hl': ('tf32', ('hh', 'hl')),
            'TF32 lh+hl': ('tf32', ('lh', 'hl')), '1xFP16': ('f16', ('hh',)), 'FP16 hh+lh': ('f16', ('hh', 'lh')),
            'FP16 hh+hl': ('f16', ('hh', 'hl')), 'FP16 lh+hl': ('f16', ('lh', 'hl'))}


@pytest.mark.parametrize('D,cin,cout', [(3, 32, 32), (3, 64, 64), (3, 256, 64), (6, 64, 32), (6, 256, 32)])
def test_criterion_separates_the_modes(D, cin, cout):
  c = _coords(cin + D, 3000, D, 10 if D == 3 else 3)
  n = len(c)
  b = so.kernel_map(c, c, so.kernel_offsets(3, D, 1))
  g = torch.Generator().manual_seed(D + cin)
  x, W = torch.randn(n, cin, generator=g), torch.randn(3 ** D, cin, cout, generator=g) / np.sqrt(cin * 8)
  ref, A = pr.conv64(x, W, b, n)
  e32 = pr.err(so.conv_forward(x, W, b, n), ref, A)
  floor = pr.f16_floor(x, W, b, n)
  for split in ('tf32', 'f16'):
    e = pr.err(pr.conv_emulated(x, W, b, n, split), ref, A, floor if split == 'f16' else None)
    assert e <= pr.bound(e32), (split, e, e32)
  for name, (split, products) in VARIANTS.items():
    e = pr.err(pr.conv_emulated(x, W, b, n, split, products), ref, A, floor if split == 'f16' else None)
    assert e >= 10 * pr.bound(e32), f'{name}: e {e:.3e} is not 10x above the bound {pr.bound(e32):.3e}'


def test_f16_floor_is_needed_and_sufficient():
  """Outputs whose only terms come from rows 2^-20 below the input maximum lose lo bits: the emulated 3xFP16 result
  misses the bare criterion there and meets it once the documented floor is subtracted."""
  n, cin, cout = 2000, 64, 32
  g = np.random.default_rng(2)
  b = [(g.permutation(n), np.arange(n))]          # one pair per output row
  t = torch.Generator().manual_seed(2)
  x, W = torch.randn(n, cin, generator=t), torch.randn(1, cin, cout, generator=t) / 8
  x[1::2] *= 2.0 ** -20
  ref, A = pr.conv64(x, W, b, n)
  e32 = pr.err(so.conv_forward(x, W, b, n), ref, A)
  X = pr.conv_emulated(x, W, b, n, 'f16')
  assert pr.err(X, ref, A) > pr.bound(e32)
  assert pr.err(X, ref, A, pr.f16_floor(x, W, b, n)) <= pr.bound(e32)
