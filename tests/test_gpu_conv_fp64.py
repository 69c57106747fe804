"""The sparse-convolution and dense-layer kernels against an fp64 reference, at their tile, chunk and padding edges.

Every kernel is held to the criterion of oracle/precision.py: e(kernel) <= KAPPA * e(fp32 oracle), with
e(X) = max |X - ref| / (A + tiny), ref and A the fp64 sum of the terms and of their absolute values.  The
3-pass tensor-core modes must meet it; their 1-pass mode on the same data must not (a negative control that
shows, on every run, that the bound sees lost bits), and is held only to its own TF32 bound.

Pair lists are either built here, with bucket sizes on the 128-row tile edges and empty buckets in between
(out rows unique and ascending inside a bucket, as the planner produces them), or taken from CoordinateManager
maps (stride 1, stride 2, transposed; D = 3 and 6).  Every test prints `RATIO <family> <case>` lines:
e(kernel) / max(e(fp32), E32_MIN), the numbers KAPPA is calibrated on.
"""
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import precision as pr
from oracle import resunet as orn
from oracle import sparse_ops as so

pytestmark = pytest.mark.gpu

# bucket sizes of the constructed maps: 1, 127, 128, 129, 255, 256, 257 pairs, empty buckets between full ones
SIZES = (0, 1, 127, 128, 129, 0, 255, 256, 257, 1000, 0, 0, 2, 63, 300, 511, 512, 513, 3, 0, 130, 126, 7, 384, 0,
         385, 33)
N_ROWS = 3000


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


def _check(family, case, X, ref, A, e32, floor=None):
  """Assert the criterion; print the ratio it is calibrated on."""
  e = pr.err(X, ref, A, floor)
  print(f'RATIO {family} {case}: e {e:.3e} e32 {e32:.3e} ratio {pr.ratio(e, e32):.3f}')
  assert e <= pr.bound(e32), f'{family} {case}: e {e:.3e} > {pr.KAPPA} * max(e32 {e32:.3e}, 2^-24)'
  return e


def _buckets(sizes, n_in, n_out, seed):
  """Pair lists with the given bucket sizes: distinct ascending out rows and distinct in rows per bucket."""
  g = np.random.default_rng(seed)
  out = []
  for s in sizes:
    s = min(s, n_in, n_out)
    out.append((g.choice(n_in, s, replace=False).astype(np.int64), np.sort(g.choice(n_out, s, replace=False))))
  return out


def _kmap(abi, buckets, n_in, n_out, pair):
  """A kernel map the _abi helpers accept as `km`, over the given pair lists, with the plain (pair=0) or the
  paired (pair=1: an even tile count per offset, padding tiles with rows <= 0) tile list of dgr_kernel_map_tiles."""
  K = len(buckets)
  kofs_h = np.concatenate([[0], np.cumsum([len(i) for i, _ in buckets])]).astype(np.int32)
  P = int(kofs_h[-1])
  per_k = (np.diff(kofs_h) + abi.TILE_ROWS - 1) // abi.TILE_ROWS
  n_tiles = int(((per_k + 1) // 2 * 2).sum() if pair else per_k.sum())
  cat = lambda k: np.concatenate([b[k] for b in buckets] + [np.zeros(1, np.int64)]).astype(np.int32)
  km = types.SimpleNamespace(K=K, n_in=n_in, n_out=n_out, nbr=None, n_pairs=P, kofs_host=kofs_h, n_tiles=n_tiles,
                             in_idx=torch.from_numpy(cat(0)).cuda(), out_idx=torch.from_numpy(cat(1)).cuda(),
                             kofs=torch.from_numpy(kofs_h).cuda())
  km.tile_k = torch.full((max(n_tiles, 1),), -1, dtype=torch.int32, device='cuda')
  km.tile_start = torch.full((max(n_tiles, 1),), -1, dtype=torch.int32, device='cuda')
  abi.call('dgr_kernel_map_tiles', abi.ptr(km.kofs), K, abi.TILE_ROWS, n_tiles, int(pair), abi.ptr(km.tile_k),
           abi.ptr(km.tile_start), abi.stream())
  return km


def _buckets_of(km):
  ii, jj, k = km.in_idx.cpu().numpy().astype(np.int64), km.out_idx.cpu().numpy().astype(np.int64), km.kofs_host
  return [(ii[k[a]:k[a + 1]], jj[k[a]:k[a + 1]]) for a in range(km.K)]


@pytest.fixture(scope='module')
def cmap(abi):
  """(buckets, plain km, paired km) of a constructed 27-offset map over 3000 rows."""
  b = _buckets(SIZES, N_ROWS, N_ROWS, seed=1)
  return b, _kmap(abi, b, N_ROWS, N_ROWS, False), _kmap(abi, b, N_ROWS, N_ROWS, True)


def _cloud(D, n, ext, seed):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-ext, ext, size=(n, D)), axis=0)
  c = c[g.permutation(len(c))]
  return np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)


@pytest.fixture(scope='module', params=[3, 6])
def real_maps(abi, request):
  """[(name, km, buckets)] of a CoordinateManager over a ~3k-row cloud: stride 1, stride 2 and its transpose."""
  from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey
  D = request.param
  man = CoordinateManager(torch.from_numpy(_cloud(D, 3000, 10 if D == 3 else 3, seed=D)).cuda())
  _, k1 = man.kernel_map(CoordinateMapKey(1), 1, 3)
  key2, k2 = man.kernel_map(CoordinateMapKey(1), 2, 3)
  _, kt = man.transpose_kernel_map(key2, 2, 3)
  return D, [(f'D{D}-{name}', km, _buckets_of(km)) for name, km in (('s1', k1), ('s2', k2), ('tr', kt))]


def _data(n, cin, K, cout, seed):
  g = torch.Generator().manual_seed(seed)
  return torch.randn(n, cin, generator=g), torch.randn(K, cin, cout, generator=g) / np.sqrt(cin * 8)


def _refs(feat, W, buckets, n_out):
  ref, A = pr.conv64(feat, W, buckets, n_out)
  return ref, A, pr.err(so.conv_forward(feat, W, buckets, n_out), ref, A)


def _tc(abi, feat, Wt, km, passes):
  out = torch.zeros(km.n_out, Wt.shape[3], device='cuda')
  abi.spconv_tc_fwd(feat, Wt, km, out, passes=passes)
  return out


# --------------------------------------------------------------------------- #
# FFMA gather-GEMM-scatter
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('cin', [1, 3, 5, 32, 36, 67])
def test_spconv_ffma_constructed(abi, cmap, cin):
  """Both column tiles (TN 32 / 64, several column blocks at cout 65, 130), the aligned (cin % 4 == 0) and scalar
  gathers, one and several 32-channel chunks, with and without the fused input ReLU."""
  b, km, _ = cmap
  for cout in (1, 3, 4, 31, 32, 33, 64, 65, 130):
    feat, W = _data(N_ROWS, cin, len(b), cout, seed=cin * 1000 + cout)
    fd, Wd = feat.cuda(), W.cuda()
    for relu_in in (False, True):
      x = torch.relu(feat) if relu_in else feat
      ref, A, e32 = _refs(x, W, b, N_ROWS)
      out = abi.spconv_fwd(fd, Wd, km, torch.zeros(N_ROWS, cout, device='cuda'), relu_in=relu_in)
      _check('ffma', f'cin{cin} cout{cout} relu{int(relu_in)}', out, ref, A, e32)


# --------------------------------------------------------------------------- #
# tensor cores: 3xTF32 / 1xTF32 and 3xFP16
# --------------------------------------------------------------------------- #
def _tf32_modes(abi, feat, W, kms, b, case, refs):
  """3xTF32 meets the criterion; 1xTF32 on the same data meets only its own TF32 bound and fails the criterion."""
  ref, A, e32 = refs
  fd, Wt = feat.cuda(), abi.pack_weight_tf32(W.cuda(), len(b), W.shape[1], W.shape[2])
  for name, km in kms:
    _check('3xtf32', f'{case} {name}', _tc(abi, fd, Wt, km, 3), ref, A, e32)
    e1 = pr.err(_tc(abi, fd, Wt, km, 1), ref, A)
    print(f'RATIO 1xtf32 {case} {name}: e {e1:.3e} e32 {e32:.3e} ratio {pr.ratio(e1, e32):.3f} '
          f'(must exceed {pr.KAPPA})')
    assert e1 <= pr.TF32_1PASS_BOUND, (case, name, e1)
    assert e1 > pr.bound(e32), f'{case} {name}: 1xTF32 passes the 3-pass criterion (e {e1:.3e}, e32 {e32:.3e})'


@pytest.mark.parametrize('cin', [32, 96, 256])
def test_spconv_tf32_constructed(abi, cmap, cin):
  """Every accumulator width, exact and padded (NT = 32 / 64 / 128 / 256), 1, 3 and 8 channel chunks, on the plain
  and the paired tile list."""
  b, km, kp = cmap
  for cout in (16, 32, 48, 64, 80, 128, 144, 256):
    feat, W = _data(N_ROWS, cin, len(b), cout, seed=cin * 1000 + cout)
    _tf32_modes(abi, feat, W, (('plain', km), ('paired', kp)), b, f'cin{cin} cout{cout}', _refs(feat, W, b, N_ROWS))


def _f16(abi, feat, W, km, amax=None):
  return abi.spconv_tc_f16_fwd(feat.cuda(), W.cuda(), km, torch.zeros(km.n_out, W.shape[2], device='cuda'),
                               amax=None if amax is None else torch.tensor([amax], dtype=torch.float32, device='cuda'))


@pytest.mark.parametrize('cin', [64, 192, 256])
def test_spconv_f16_constructed(abi, cmap, cin):
  """3xFP16 at every accumulator width (NT = 32 / 64 / 128 / 256, exact and padded) and 1, 3, 4 chunks."""
  b, km, kp = cmap
  for cout in (32, 64, 96, 128, 160, 256):
    feat, W = _data(N_ROWS, cin, len(b), cout, seed=cin * 1000 + cout + 7)
    ref, A, e32 = _refs(feat, W, b, N_ROWS)
    floor = pr.f16_floor(feat, W, b, N_ROWS)
    for name, m in (('plain', km), ('paired', kp)):
      _check('3xfp16', f'cin{cin} cout{cout} {name}', _f16(abi, feat, W, m), ref, A, e32, floor)


def test_spconv_f16_oversized_amax_fails(abi, cmap):
  """Negative control: amax is documented as an upper bound, but one 2^20 too large pushes every input element below
  fp16's normal range and loses bits far beyond the documented floor: the criterion must see it."""
  b, km, _ = cmap
  for cout in (32, 64):
    feat, W = _data(N_ROWS, 64, len(b), cout, seed=cout + 11)
    ref, A, e32 = _refs(feat, W, b, N_ROWS)
    floor = pr.f16_floor(feat, W, b, N_ROWS)
    amax = float(feat.abs().max())
    _check('3xfp16', f'amax-exact cout{cout}', _f16(abi, feat, W, km, amax), ref, A, e32, floor)
    e = pr.err(_f16(abi, feat, W, km, amax * 2.0 ** 20), ref, A, floor)
    print(f'RATIO 3xfp16-amax2^20 cout{cout}: e {e:.3e} e32 {e32:.3e} ratio {pr.ratio(e, e32):.3f} '
          f'(must exceed {pr.KAPPA})')
    assert e > pr.bound(e32), f'an amax 2^20 too large passes the criterion (e {e:.3e}, e32 {e32:.3e})'


def test_spconv_f16_data_edges(abi, cmap):
  b, km, _ = cmap
  K, cin, cout = len(b), 128, 64
  feat, W = _data(N_ROWS, cin, K, cout, seed=21)
  # all-zero input: exactly zero output (amax 0 selects the unit scale)
  z = _f16(abi, torch.zeros(N_ROWS, cin), W, km)
  assert torch.equal(z, torch.zeros_like(z))
  ref, A, e32 = _refs(feat, W, b, N_ROWS)
  floor = pr.f16_floor(feat, W, b, N_ROWS)
  amax = float(feat.abs().max())
  for loose in (2.0, 2.0 ** 6):          # amax as a loose upper bound
    _check('3xfp16', f'amax x{loose:g}', _f16(abi, feat, W, km, amax * loose), ref, A, e32, floor)
  # rows 2^-20 below the maximum: within the documented floor
  small = feat.clone()
  small[1::3] *= 2.0 ** -20
  ref, A, e32 = _refs(small, W, b, N_ROWS)
  _check('3xfp16', 'rows 2^-20', _f16(abi, small, W, km), ref, A, e32, pr.f16_floor(small, W, b, N_ROWS))
  # one weight outlier sets the weight scale: every other weight sits 2^10..2^20 below it
  Wo = W.clone()
  Wo[9, 5, 17] = 1000.0
  ref, A, e32 = _refs(feat, Wo, b, N_ROWS)
  _check('3xfp16', 'weight outlier', _f16(abi, feat, Wo, km), ref, A, e32, pr.f16_floor(feat, Wo, b, N_ROWS))
  # amax exactly a power of two (the scale maps it to 2^14 exactly)
  p2 = (feat / feat.abs().max() * 3.9).clamp(-3.9, 3.9)
  p2[7, 3] = -4.0
  ref, A, e32 = _refs(p2, W, b, N_ROWS)
  assert float(p2.abs().max()) == 4.0
  _check('3xfp16', 'amax 2^2', _f16(abi, p2, W, km), ref, A, e32, pr.f16_floor(p2, W, b, N_ROWS))


def test_packed_weights_equal_emulated_splits(abi):
  """The packed TF32 and fp16 weight slabs hold exactly the splits oracle/precision.py emulates (same rounding)."""
  K, cin, cout = 3, 128, 64
  g = torch.Generator().manual_seed(3)
  W = torch.randn(K, cin, cout, generator=g) * torch.exp(4 * torch.randn(K, cin, cout, generator=g))
  # TF32 ties (round to nearest even would go the other way on each) and signed zeros
  W[0, 0, :6] = torch.tensor([1 + 2 ** -11, -(1 + 2 ** -11), 1 + 5 * 2 ** -11, -(1 + 5 * 2 ** -11), 0.0, -0.0])
  n = torch.arange(cout)

  def unswizzle(t, q_pieces):         # [K, chunks, 2, cout, q_pieces * w] pieces XOR-swizzled by (row & 7)
    w = t.shape[-1] // 8
    out = torch.empty_like(t)
    for q in range(8):
      src = (q ^ (n & 7))
      for r in range(cout):
        out[..., r, w * q:w * q + w] = t[..., r, w * int(src[r]):w * int(src[r]) + w]
    return out

  pk = unswizzle(abi.pack_weight_tf32(W.cuda().contiguous(), K, cin, cout).cpu(), 8)
  hi, lo = pr.tf32_split(W.numpy())
  to_pk = lambda a: torch.from_numpy(a).reshape(K, cin // 32, 32, cout).permute(0, 1, 3, 2)
  assert torch.equal(pk[:, :, 0].contiguous().view(torch.int32), to_pk(hi).contiguous().view(torch.int32))
  assert torch.equal(pk[:, :, 1].contiguous().view(torch.int32), to_pk(lo).contiguous().view(torch.int32))
  packed = torch.empty(4 * K * cin * cout, dtype=torch.uint8, device='cuda')
  wscale = torch.empty(2, dtype=torch.float32, device='cuda')
  Wd = W.cuda().contiguous()
  abi.call('dgr_pack_weight_f16', abi.ptr(Wd), K, cin, cout, abi.ptr(packed), abi.ptr(wscale), abi.stream())
  pf = unswizzle(packed.cpu().view(torch.int16).reshape(K, cin // 64, 2, cout, 64), 8)
  fh, fl, s = pr.f16_split(W.numpy())
  to_pf = lambda a: torch.from_numpy(a.view(np.int16)).reshape(K, cin // 64, 64, cout).permute(0, 1, 3, 2)
  assert torch.equal(pf[:, :, 0], to_pf(fh).contiguous())
  assert torch.equal(pf[:, :, 1], to_pf(fl).contiguous())
  assert float(wscale[0]) == 1.0 / float(s) and float(wscale[1]) == float(W.abs().max())


# --------------------------------------------------------------------------- #
# every mode on CoordinateManager maps
# --------------------------------------------------------------------------- #
def test_all_modes_on_real_maps(abi, real_maps):
  D, maps = real_maps
  for name, km, b in maps:
    for cin, cout in ((64, 64), (128, 32)):
      feat, W = _data(km.n_in, cin, km.K, cout, seed=cin + cout + D)
      ref, A, e32 = _refs(feat, W, b, km.n_out)
      fd, Wd = feat.cuda(), W.cuda()
      out = abi.spconv_fwd(fd, Wd, km, torch.zeros(km.n_out, cout, device='cuda'))
      _check('ffma', f'{name} {cin}->{cout}', out, ref, A, e32)
      _tf32_modes(abi, feat, W, (('plain', km),), b, f'{name} {cin}->{cout}', (ref, A, e32))
      _check('3xfp16', f'{name} {cin}->{cout}', _f16(abi, feat, W, km), ref, A, e32, pr.f16_floor(feat, W, b, km.n_out))


# --------------------------------------------------------------------------- #
# conv1 kernels: neighbour table and occupancy bits
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('K', [125, 343])
def test_table_and_ones_bits(abi, K):
  """The table kernel for every cin 1..8 and cout 16 / 32 / 64 (weight chunks of kc_max offsets, kc_max % 8 != 0 at
  cin 4..8, cout 64), on a neighbour table whose row stride exceeds its row count; the ones-bits kernel (several
  weight chunks at cout 64, K 343) bit-identical to the table kernel on an all-ones input; both against fp64."""
  n, stride = N_ROWS, N_ROWS + 37
  b = _buckets([SIZES[k % len(SIZES)] for k in range(K)], n, n, seed=K)
  nbr_h = np.zeros((K, stride), np.int32)       # padding columns: a valid row, so a read of them would show
  nbr_h[:, :n] = -1
  bits_h = np.zeros((K, (n + 31) // 32), np.uint32)
  for k, (i, j) in enumerate(b):
    nbr_h[k, j] = i
    np.bitwise_or.at(bits_h[k], j >> 5, (np.uint32(1) << (j & 31).astype(np.uint32)))
  km = types.SimpleNamespace(K=K, n_out=n, nbr=torch.from_numpy(nbr_h).cuda()[:, :n])
  assert km.nbr.stride(0) == stride
  bits = torch.from_numpy(bits_h.view(np.int32)).cuda()
  g = torch.Generator().manual_seed(K)
  for cout in (16, 32, 64):
    scale, shift = torch.rand(cout, generator=g) + 0.5, torch.randn(cout, generator=g)
    sd, hd = scale.cuda(), shift.cuda()
    for cin in range(1, 9):
      feat, W = _data(n, cin, K, cout, seed=K + 10 * cin + cout)
      ref, A = pr.conv64(feat, W, b, n)
      e32 = pr.err(so.conv_forward(feat, W, b, n), ref, A)
      Wd = W.cuda().contiguous()
      _check('table', f'K{K} cin{cin} cout{cout}', abi.spconv_table_fwd(feat.cuda(), Wd, km, cout), ref, A, e32)
      # fused BatchNorm epilogue: out * scale + shift
      s64, h64 = scale.double().numpy(), shift.double().numpy()
      e32s = pr.err(so.conv_forward(feat, W, b, n) * scale + shift, ref * s64 + h64, A * np.abs(s64) + np.abs(h64))
      got = abi.spconv_table_fwd(feat.cuda(), Wd, km, cout, sd, hd)
      _check('table', f'K{K} cin{cin} cout{cout} bn', got, ref * s64 + h64, A * np.abs(s64) + np.abs(h64), e32s)
    W1 = _data(n, 1, K, cout, seed=K + cout)[1]
    ones, W1d = torch.ones(n, 1), W1.cuda()
    want = abi.spconv_table_fwd(ones.cuda(), W1d, km, cout, sd, hd)
    got = torch.empty(n, cout, device='cuda')
    abi.call('dgr_spconv_ones_bits_fwd', abi.ptr(W1d), cout, abi.ptr(bits), bits_h.shape[1], K, n, abi.ptr(sd),
             abi.ptr(hd), abi.ptr(got), abi.stream())
    assert torch.equal(got, want), f'ones-bits != table, K {K} cout {cout}'
    ref, A = pr.conv64(ones, W1, b, n)
    s64, h64 = scale.double().numpy(), shift.double().numpy()
    e32 = pr.err(so.conv_forward(ones, W1, b, n) * scale + shift, ref * s64 + h64, A * np.abs(s64) + np.abs(h64))
    _check('ones-bits', f'K{K} cout{cout}', got, ref * s64 + h64, A * np.abs(s64) + np.abs(h64), e32)


# --------------------------------------------------------------------------- #
# dense layers
# --------------------------------------------------------------------------- #
def _normalized(v, A, xp):
  """Row-normalised v / (|v| + 1e-8) and its term magnitude A / (|v| + 1e-8)."""
  den = xp.sqrt((v * v).sum(1, keepdims=True)) + 1e-8
  return v / den, A / den


@pytest.mark.parametrize('ca,cb', [(64, 32), (5, 0), (6, 3), (33, 31)])
def test_linear_fwd(abi, ca, cb):
  """1x1 convolution with the fused concat, bias, ReLU and row normalisation: one and several column blocks,
  scalar and vector loads and stores, tile-edge row counts, all-zero rows."""
  g = torch.Generator().manual_seed(ca + cb)
  for cout in (1, 3, 32, 33, 64, 65, 130):
    for n in (1, 127, 128, 129, 1000):
      a = torch.randn(n, ca, generator=g)
      b = torch.randn(n, cb, generator=g) if cb else None
      a[n // 2] = 0
      if cb:
        b[n // 2] = 0
      W = torch.randn(ca + cb, cout, generator=g) / np.sqrt(ca + cb)
      bias = torch.randn(cout, generator=g)
      x32 = a if b is None else torch.cat([a, b], 1)
      args = (a.cuda(), W.cuda())
      for use_bias, relu, norm in ((False, False, False), (True, True, False), (False, False, True),
                                   (True, False, True)):
        if norm and cout > 64:
          continue
        bb = bias if use_bias else None
        ref, A = pr.linear64(a, W, bb, b)
        y32 = so.linear_forward(x32, W, bb)
        if relu:
          ref, y32 = np.maximum(ref, 0), torch.relu(y32)
        if norm:
          y32 = y32 / (torch.norm(y32, dim=1, keepdim=True) + 1e-8)
          ref, A = _normalized(ref, A, np)
        got = abi.linear_fwd(*args, None if bb is None else bb.cuda(), b=None if b is None else b.cuda(), relu=relu,
                             normalize=norm)
        _check('linear', f'{ca}+{cb}->{cout} n{n} bias{int(use_bias)} relu{int(relu)} norm{int(norm)}', got, ref, A,
               pr.err(y32, ref, A))
        if norm and not use_bias:
          assert not got[n // 2].any(), 'an all-zero row must normalise to zero'


def _affine_ref(x, s, h, r, relu):
  ref = x.double().numpy()
  A = np.abs(ref)
  if s is not None:
    ref = ref * s.double().numpy() + h.double().numpy()
    A = A * np.abs(s.double().numpy()) + np.abs(h.double().numpy())
  if r is not None:
    ref, A = ref + r.double().numpy(), A + np.abs(r.double().numpy())
  y = x if s is None else x * s + h
  y = y if r is None else y + r
  return (np.maximum(ref, 0) if relu else ref), A, (torch.relu(y) if relu else y)


@pytest.mark.parametrize('c', [1, 3, 6, 64, 130])
def test_affine_act(abi, c):
  """Scale / shift, residual, ReLU on the float4 path (c % 4 == 0, with its amax slot) and the scalar path."""
  g = torch.Generator().manual_seed(c)
  n = 1000
  x = torch.randn(n, c, generator=g) * 3
  s, h, r = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g), torch.randn(n, c, generator=g)
  for use_s in (False, True):
    for use_r in (False, True):
      for relu in (False, True):
        ss, rr = (s, h) if use_s else (None, None), r if use_r else None
        ref, A, y32 = _affine_ref(x, *ss, rr, relu)
        dev = [None if t is None else t.cuda() for t in (x, *ss, rr)]
        out = torch.empty(n, c, device='cuda')
        amax = torch.zeros(1, device='cuda') if c % 4 == 0 else None
        abi.call('dgr_affine_act_amax', *(abi.ptr(t) for t in dev[:1]), n, c, *(abi.ptr(t) for t in dev[1:]),
                 int(relu), abi.ptr(out), abi.ptr(amax), abi.stream())
        _check('affine', f'c{c} scale{int(use_s)} res{int(use_r)} relu{int(relu)}', out, ref, A, pr.err(y32, ref, A))
        if amax is not None:
          assert float(amax) == float(out.abs().max()), 'amax slot != max |out|'


def test_affine_amax_accumulates(abi):
  """The amax slot is max |out| exactly, reduced over two launches into one slot (the caller zeroes it), with negative
  values that dominate before the ReLU and without it."""
  g = torch.Generator().manual_seed(5)
  x1, x2 = torch.randn(777, 64, generator=g), torch.randn(3001, 64, generator=g)
  x2[123, 7] = -50.0                                   # the largest magnitude is negative
  x1[5, 3] = 20.0
  for relu in (False, True):
    slot = torch.zeros(1, device='cuda')
    outs = []
    for x in (x1.cuda(), x2.cuda()):
      out = torch.empty_like(x)
      abi.call('dgr_affine_act_amax', abi.ptr(x), x.shape[0], 64, None, None, None, int(relu), abi.ptr(out),
               abi.ptr(slot), abi.stream())
      outs.append(out)
    want = max(float(o.abs().max()) for o in outs)
    assert float(slot) == want == (20.0 if relu else 50.0), (relu, float(slot), want)


@pytest.mark.parametrize('c', [1, 33, 100])
def test_cat2_and_l2_normalize(abi, c):
  g = torch.Generator().manual_seed(c)
  n = 1000
  a = torch.randn(n, c, generator=g)
  a[::7] = 0
  for cb in (1, 33, 100):
    b = torch.randn(n, cb, generator=g)
    assert torch.equal(abi.cat2(a.cuda(), b.cuda()).cpu(), torch.cat([a, b], 1))
  ref, A = _normalized(a.double().numpy(), np.abs(a.double().numpy()), np)
  got = abi.l2_normalize(a.cuda())
  _check('l2', f'c{c}', got, ref, A, pr.err(a / (a.norm(dim=1, keepdim=True) + 1e-8), ref, A))
  assert not got[::7].any()


# --------------------------------------------------------------------------- #
# weight gradient
# --------------------------------------------------------------------------- #
@pytest.mark.parametrize('cin', [1, 6, 33, 65, 100])
def test_spconv_wgrad(abi, cin):
  """dW against fp64 with channel counts that straddle the 32 / 64 blocks, empty buckets and buckets longer than the
  32-pair stage; dw starts as NaN, so every entry is shown to be written."""
  n = 1500
  b = _buckets((0, 1, 31, 32, 33, 0, 64, 65, 200, 0, 1000, 7), n, n, seed=cin)
  km = _kmap(abi, b, n, n, False)
  for cout in (1, 6, 33, 65, 100):
    feat, gout = _data(n, cin, 1, cout, seed=cin * 100 + cout)[0], _data(n, cout, 1, 1, seed=cout)[0]
    ref, A = pr.wgrad64(feat, gout, b)
    dw = torch.full((km.K, cin, cout), float('nan'), device='cuda')
    fd, gd = feat.cuda(), gout.cuda()
    abi.call('dgr_spconv_wgrad', abi.ptr(fd), cin, abi.ptr(gd), cout, abi.ptr(km.in_idx), abi.ptr(km.out_idx),
             abi.ptr(km.kofs), km.K, abi.ptr(dw), abi.stream())
    assert bool(torch.isfinite(dw).all())
    for k, (i, _) in enumerate(b):
      if len(i) == 0:
        assert not dw[k].any()
    _check('wgrad', f'cin{cin} cout{cout}', dw, ref, A, pr.err(pr.wgrad32(feat, gout, b), ref, A))


# --------------------------------------------------------------------------- #
# malformed input: rejected before any launch
# --------------------------------------------------------------------------- #
def test_argument_checks(abi):
  f = torch.zeros(256, 64, device='cuda')
  i = torch.zeros(8, dtype=torch.int32, device='cuda')
  P, s = abi.ptr, abi.stream()
  bad = [
      ('dgr_spconv_fwd', P(f), 64, P(f), 64, P(i), P(i), P(i), P(i), P(i), 1, 64, 0, P(f), s),           # tile rows
      ('dgr_spconv_tc_fwd', P(f), 64, P(f), 64, P(i), P(i), P(i), P(i), P(i), 1, 128, 2, P(f), s),       # passes
      ('dgr_spconv_tc_fwd', P(f), 64, P(f), 8, P(i), P(i), P(i), P(i), P(i), 1, 128, 3, P(f), s),        # cout 8
      ('dgr_spconv_tc_f16_fwd', P(f), 32, P(f), 64, P(i), P(i), P(i), P(i), P(i), 1, 128, P(f), P(f), P(f), s),
      ('dgr_spconv_tc_f16_fwd', P(f), 64, P(f), 64, P(i), P(i), P(i), P(i), P(i), 1, 128, None, P(f), P(f), s),
      ('dgr_spconv_table_fwd_strided', P(f), 9, P(f), 32, P(i), 27, 8, 8, None, None, P(f), s),            # cin 9
      ('dgr_spconv_table_fwd_strided', P(f), 4, P(f), 32, P(i), 27, 8, 7, None, None, P(f), s),            # stride
      ('dgr_spconv_table_fwd_strided', P(f), 4, P(f), 48, P(i), 27, 8, 8, None, None, P(f), s),            # cout 48
      ('dgr_spconv_ones_bits_fwd', P(f), 32, P(i), 1, 27, 33, None, None, P(f), s),                       # mask words
      ('dgr_linear_fwd', P(f), 64, None, 0, 8, P(f), 65, None, 0, 1, P(f), s),                            # normalize
      ('dgr_affine_act_amax', P(f), 8, 6, None, None, None, 0, P(f), P(f), s),                            # amax c % 4
      ('dgr_affine_act_amax', P(f), 8, 8, P(f), None, None, 0, P(f), None, s),                            # scale only
      ('dgr_spconv_wgrad', P(f), 64, P(f), 64, P(i), P(i), P(i), 0, P(f), s),                             # K 0
  ]
  before = f.clone()
  for name, *args in bad:
    with pytest.raises(abi.DgrError):
      abi.call(name, *args)
  torch.cuda.synchronize()
  assert torch.equal(f, before)


# --------------------------------------------------------------------------- #
# end to end: the whole network against its fp64 forward
# --------------------------------------------------------------------------- #
# The per-layer excess of the tensor-core layers over an fp32 computation (up to KAPPA) compounds over the 22 layers of
# the network.  Measured on one H100 80GB HBM3 (400 W), rms distance from fp64 over the fp32 oracle's: FCGF native 6.4,
# FCGF operator path 8.9, 6-D inlier net 1.2 (both paths).
KAPPA_NET = 16.0


@pytest.mark.parametrize('which', ['fcgf', 'inlier'])
def test_network_against_fp64(abi, which):
  """The native executor (its real mix of bits / table / 3xFP16 / 3xTF32 layers and fused epilogues) and the operator
  path against oracle.resunet in fp64, on ~10k voxels: their distance from fp64 no larger than KAPPA_NET times the
  fp32 oracle's own."""
  from deepglobalregistration_b200 import me as ME, native
  from deepglobalregistration_b200.model import load_model
  xyz = syn.room_scan(0 if which == 'fcgf' else 1, n_raw=20000, extent=(1.8, 1.5, 1.25))
  c0 = so.batched_coordinates([so.quantize_first(xyz, 0.05)[0]])
  if which == 'fcgf':
    sd, coords, args = syn.make_checkpoint(0, with_inlier=False)['state_dict'], c0, (7, True)
    model = load_model('ResUNetBN2C')(1, 32, bn_momentum=0.05, conv1_kernel_size=7, normalize_feature=True)
  else:
    g = np.random.default_rng(0)
    c1 = c0[:, 1:] + np.array([3, -2, 1])
    rnd = g.random(len(c0)) < 0.6
    c1[rnd] = c0[g.integers(0, len(c0), int(rnd.sum())), 1:]
    coords = np.concatenate([c0, c1], 1).astype(np.int32)
    sd, args = syn.resunet_state_dict(5, 1, 1, 3, 6), (3, False)
    model = load_model('ResUNetBN2C')(1, 1, bn_momentum=0.05, conv1_kernel_size=3, normalize_feature=False, D=6)
  assert len(coords) > 8000
  ones = torch.ones(len(coords), 1)
  ref = orn.resunet_forward(sd, coords, ones, *args, dtype=torch.float64).numpy()
  # distance from fp64: root mean square over every output (the maximum of an error compounded over 22 layers is
  # one sample of a heavy tail; it is printed beside)
  rms = lambda X: float(np.sqrt(((X.detach().cpu().double().numpy() - ref) ** 2).mean()))
  mx = lambda X: float(np.abs(X.detach().cpu().double().numpy() - ref).max())
  r32 = orn.resunet_forward(sd, coords, ones, *args)
  e32, m32 = rms(r32), mx(r32)
  model.load_state_dict(sd)
  model = model.cuda().eval()
  ct = torch.from_numpy(coords).cuda().contiguous()
  net, ctx = native.Net(model, 'cuda'), native.Context('cuda')
  try:
    got = {'native': net.forward(ctx, ct)}
  finally:
    net.close()
    ctx.close()
  with torch.no_grad():
    got['operator'] = model(ME.SparseTensor(ones, coordinates=ct, device='cuda')).F
  for path, X in got.items():
    e = rms(X)
    print(f'RATIO network {which} {path}: e {e:.3e} e32 {e32:.3e} ratio {e / e32:.3f} '
          f'(max |X - ref64| {mx(X):.3e}, fp32 oracle {m32:.3e})')
    assert e <= KAPPA_NET * e32, f'{which} {path}: rms {e:.3e} > {KAPPA_NET} * {e32:.3e}'
