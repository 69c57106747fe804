"""GPU parity of the sparse convolution and dense layers against the oracle (fp32).

Tolerance: the CUDA kernels and the oracle both accumulate in fp32 but in different
orders (per-offset scatter-add with atomics vs ascending-kappa index_add), so results
agree to a few ulp of the accumulated magnitude: |diff| <= 2e-5 * (1 + |ref|) here; an
fp64 oracle pass bounds the fp32 oracle's own rounding at the same level."""
import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import resunet as orn
from oracle import sparse_ops as so

pytestmark = pytest.mark.gpu
RTOL = 2e-5


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


def _close(got, want, tol=RTOL, what=''):
  got, want = got.detach().cpu().double(), want.detach().cpu().double()
  assert got.shape == want.shape, (what, got.shape, want.shape)
  err = (got - want).abs() / (1 + want.abs())
  assert float(err.max()) <= tol, f'{what}: max rel err {float(err.max()):.3e}'


def _coords(seed, n, D, span):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-span, span, size=(n, D)), axis=0)
  c = c[g.permutation(len(c))]
  return np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)


@pytest.mark.parametrize('D,cin,cout,ks', [(3, 32, 32, 3), (3, 32, 64, 3), (3, 64, 128, 3), (3, 256, 128, 3),
                                           (3, 96, 40, 3), (3, 1, 32, 7), (3, 3, 32, 5), (3, 6, 16, 3),
                                           (6, 1, 32, 3), (6, 6, 32, 3), (6, 32, 32, 3), (6, 64, 64, 3)])
def test_spconv_stride1(abi, D, cin, cout, ks):
  from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey
  coords = _coords(cin + cout + D, 2500, D, 10 if D == 3 else 3)
  n = len(coords)
  g = torch.Generator().manual_seed(1)
  feat = torch.randn(n, cin, generator=g)
  W = torch.randn(ks ** D, cin, cout, generator=g) / np.sqrt(cin * 8)
  man = CoordinateManager(torch.from_numpy(coords).cuda())
  _, km = man.kernel_map(CoordinateMapKey(1), 1, ks)
  buckets = so.kernel_map(coords, coords, so.kernel_offsets(ks, D, 1))
  want = so.conv_forward(feat, W, buckets, n)
  out = torch.zeros(n, cout, device='cuda')
  abi.spconv_fwd(feat.cuda(), W.cuda().contiguous(), km, out)
  _close(out, want, what='spconv_fwd')
  if km.nbr is not None and cin <= 8 and cout in (16, 32, 64):
    scale, shift = torch.rand(cout) + 0.5, torch.randn(cout)
    got = abi.spconv_table_fwd(feat.cuda(), W.cuda().contiguous(), km, cout, scale.cuda(), shift.cuda())
    _close(got, want * scale + shift, what='spconv_table_fwd')
  # fused input ReLU
  out2 = torch.zeros(n, cout, device='cuda')
  abi.spconv_fwd(feat.cuda(), W.cuda().contiguous(), km, out2, relu_in=True)
  _close(out2, so.conv_forward(torch.relu(feat), W, buckets, n), what='spconv_fwd relu_in')


@pytest.mark.parametrize('D,cin,cout', [(3, 32, 32), (3, 32, 64), (3, 64, 64), (3, 64, 128), (3, 128, 128),
                                        (3, 256, 256), (3, 256, 128), (3, 128, 64), (3, 96, 48), (6, 32, 32),
                                        (6, 256, 256), (3, 32, 16), (3, 64, 240)])
def test_spconv_tensor_core(abi, D, cin, cout):
  """wgmma path: 3xTF32 must match the fp32 oracle like the FFMA kernel does; single-pass
  TF32 within 5e-3 of the result's scale."""
  from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey
  assert abi.tc_supported(cin, cout)
  coords = _coords(3 * cin + cout + D, 3000, D, 10 if D == 3 else 3)
  n = len(coords)
  g = torch.Generator().manual_seed(4)
  feat = torch.randn(n, cin, generator=g)
  W = torch.randn(3 ** D, cin, cout, generator=g) / np.sqrt(cin * 8)
  man = CoordinateManager(torch.from_numpy(coords).cuda())
  _, km = man.kernel_map(CoordinateMapKey(1), 1, 3)
  want = so.conv_forward(feat, W, so.kernel_map(coords, coords, so.kernel_offsets(3, D, 1)), n)
  Wd = W.cuda().contiguous()
  Wt = abi.pack_weight_tf32(Wd, 3 ** D, cin, cout)
  # packed layout: [K, cin/32, (hi, lo), cout, 32] with 16-byte pieces XOR-swizzled by (row & 7)
  pk = Wt.cpu()
  hi = pk[:, :, 0] + pk[:, :, 1]                       # hi + lo == the fp32 weight, exactly
  n_idx = torch.arange(cout)
  unsw = torch.empty_like(hi)
  for q in range(8):
    src_piece = (q ^ (n_idx & 7))
    for nn in range(cout):
      unsw[:, :, nn, 4 * q:4 * q + 4] = hi[:, :, nn, 4 * int(src_piece[nn]):4 * int(src_piece[nn]) + 4]
  want_w = W.reshape(3 ** D, cin // 32, 32, cout).permute(0, 1, 3, 2)
  assert torch.equal(unsw, want_w)
  out = torch.zeros(n, cout, device='cuda')
  abi.spconv_tc_fwd(feat.cuda(), Wt, km, out, passes=3)
  _close(out, want, what='wgmma 3xTF32')
  out1 = torch.zeros(n, cout, device='cuda')
  abi.spconv_tc_fwd(feat.cuda(), Wt, km, out1, passes=1)
  scale = float(want.abs().max())
  assert float((out1.cpu() - want).abs().max()) <= 5e-3 * scale, 'wgmma 1xTF32'
  # accumulate onto a non-zero initial value, twice in a row (persistent CTAs, phase tracking)
  init = torch.randn(n, cout, generator=g)
  out2 = init.clone().cuda()
  abi.spconv_tc_fwd(feat.cuda(), Wt, km, out2, passes=3)
  abi.spconv_tc_fwd(feat.cuda(), Wt, km, out2, passes=3)
  _close(out2, init + 2 * want, what='wgmma accumulate')


@pytest.mark.parametrize('D,cin,cout', [(3, 256, 256), (3, 128, 128), (6, 64, 240), (3, 32, 32)])
def test_spconv_tensor_core_cta_pairs(abi, D, cin, cout):
  """The tensor-core convolution on the paired tile list (an even tile count per offset, as CTA pairs consume it,
  with empty padding tiles) and on the plain one must match the oracle, run after run."""
  from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey
  coords = _coords(cin + 7 * cout + D, 4000, D, 10 if D == 3 else 3)
  n = len(coords)
  g = torch.Generator().manual_seed(5)
  feat = torch.randn(n, cin, generator=g)
  W = torch.randn(3 ** D, cin, cout, generator=g) / np.sqrt(cin * 8)
  man = CoordinateManager(torch.from_numpy(coords).cuda())
  _, km = man.kernel_map(CoordinateMapKey(1), 1, 3)
  want = so.conv_forward(feat, W, so.kernel_map(coords, coords, so.kernel_offsets(3, D, 1)), n)
  Wt = abi.pack_weight_tf32(W.cuda().contiguous(), 3 ** D, cin, cout)
  tk, ts, nt = km.paired_tiles()
  assert nt % 2 == 0 and nt >= km.n_tiles
  tkh = tk.cpu().numpy()[:nt]
  assert (tkh[0::2] == tkh[1::2]).all()              # both tiles of a pair share the kernel offset
  for (tl_k, tl_s, tl_n), name in (((tk, ts, nt), 'paired tile list'), ((km.tile_k, km.tile_start, km.n_tiles), 'plain tile list')):
    for rep in range(2):
      out = torch.zeros(n, cout, device='cuda')
      abi.call('dgr_spconv_tc_fwd', abi.ptr(feat.cuda()), cin, abi.ptr(Wt), cout, abi.ptr(km.in_idx), abi.ptr(km.out_idx),
               abi.ptr(km.kofs), abi.ptr(tl_k), abi.ptr(tl_s), tl_n, abi.TILE_ROWS, 3, abi.ptr(out), abi.stream())
      _close(out, want, what=f'wgmma {name}')


def test_tc_unsupported_shapes_fall_back(abi):
  assert not abi.tc_supported(1, 32) and not abi.tc_supported(48, 32) and not abi.tc_supported(32, 8)
  assert not abi.tc_supported(32, 264) and abi.tc_supported(64, 256)


@pytest.mark.parametrize('D,cin,cout', [(3, 32, 64), (3, 128, 256), (6, 32, 64)])
def test_spconv_stride2_and_transpose(abi, D, cin, cout):
  from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey
  coords = _coords(7 + D, 3000, D, 12 if D == 3 else 3)
  coarse, _ = so.stride_coords(coords, 2)
  nf, nc = len(coords), len(coarse)
  g = torch.Generator().manual_seed(2)
  man = CoordinateManager(torch.from_numpy(coords).cuda())
  key2, kd = man.kernel_map(CoordinateMapKey(1), 2, 3)
  down = so.kernel_map(coords, coarse, so.kernel_offsets(3, D, 1))
  feat = torch.randn(nf, cin, generator=g)
  W = torch.randn(3 ** D, cin, cout, generator=g) / np.sqrt(cin * 4)
  out = torch.zeros(nc, cout, device='cuda')
  abi.spconv_fwd(feat.cuda(), W.cuda(), kd, out)
  _close(out, so.conv_forward(feat, W, down, nc), what='stride-2 conv')
  _, kt = man.transpose_kernel_map(key2, 2, 3)
  cfeat = torch.randn(nc, cout, generator=g)
  Wt = torch.randn(3 ** D, cout, cin, generator=g) / np.sqrt(cout)
  out_t = torch.zeros(nf, cin, device='cuda')
  abi.spconv_fwd(cfeat.cuda(), Wt.cuda(), kt, out_t)
  _close(out_t, so.conv_forward(cfeat, Wt, so.swap_map(down), nf), what='transposed conv')


def test_linear_and_elementwise(abi):
  g = torch.Generator().manual_seed(3)
  n = 1000
  a, b = torch.randn(n, 64, generator=g), torch.randn(n, 32, generator=g)
  W = torch.randn(96, 64, generator=g) / 10
  _close(abi.linear_fwd(a.cuda(), W.cuda(), None, b=b.cuda(), relu=True),
         torch.relu(torch.cat([a, b], 1) @ W), what='linear cat relu')
  W2, bias = torch.randn(64, 32, generator=g) / 8, torch.randn(1, 32, generator=g)
  y = a @ W2 + bias
  _close(abi.linear_fwd(a.cuda(), W2.cuda(), bias.cuda().reshape(-1)), y, what='linear bias')
  _close(abi.linear_fwd(a.cuda(), W2.cuda(), bias.cuda().reshape(-1), normalize=True),
         y / (y.norm(dim=1, keepdim=True) + 1e-8), what='linear normalize')
  W3, b3 = torch.randn(64, 1, generator=g), torch.randn(1, 1, generator=g)
  _close(abi.linear_fwd(a.cuda(), W3.cuda(), b3.cuda().reshape(-1)), a @ W3 + b3, what='linear cout=1')
  a6 = torch.randn(n, 6, generator=g)
  W6 = torch.randn(6, 48, generator=g)
  _close(abi.linear_fwd(a6.cuda(), W6.cuda()), a6 @ W6, what='linear cin=6')
  # elementwise
  sc, sh = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g)
  r = torch.randn(n, 64, generator=g)
  _close(abi.affine_act(a.cuda(), sc.cuda(), sh.cuda(), r.cuda(), relu=True), torch.relu(a * sc + sh + r),
         tol=1e-6, what='affine_act')
  x1 = torch.randn(n, 1, generator=g)
  _close(abi.affine_act(x1.cuda(), relu=True), torch.relu(x1), tol=0, what='relu c=1')
  _close(abi.cat2(a.cuda(), b.cuda()), torch.cat([a, b], 1), tol=0, what='cat2')
  _close(abi.l2_normalize(a.cuda()), a / (a.norm(dim=1, keepdim=True) + 1e-8), tol=1e-6, what='l2')


def _small_pair_cloud(seed=0, n_raw=20000):
  xyz = syn.room_scan(seed, n_raw=n_raw, extent=(1.8, 1.5, 1.25))
  coords, sel = so.quantize_first(xyz, 0.05)
  return so.batched_coordinates([coords])


def _forward(model, coords, path):
  """The network on all-ones input: operator by operator, or on the native executor."""
  from deepglobalregistration_b200 import me as ME, native
  ct = torch.from_numpy(coords).cuda().contiguous()
  if path == 'native':
    return native.Net(model, 'cuda').forward(native.Context('cuda'), ct)
  with torch.no_grad():
    return model(ME.SparseTensor(torch.ones(len(coords), 1), coordinates=ct, device='cuda')).F


@pytest.mark.parametrize('path', ['operator', 'native'])
def test_resunet_fcgf_forward(abi, path):
  from deepglobalregistration_b200.model import load_model
  state = syn.make_checkpoint(0, with_inlier=False)
  coords = _small_pair_cloud()
  taps = {}
  want = orn.resunet_forward(state['state_dict'], coords, torch.ones(len(coords), 1), 7, True, taps=taps)
  model = load_model('ResUNetBN2C')(1, 32, bn_momentum=0.05, conv1_kernel_size=7, normalize_feature=True)
  model.load_state_dict(state['state_dict'])
  model = model.cuda().eval()
  got = _forward(model, coords, path)
  _close(got, want, tol=5e-5, what='FCGF features')
  assert torch.allclose(got.norm(dim=1).cpu(), torch.ones(len(coords)), atol=1e-5)


@pytest.mark.parametrize('path', ['operator', 'native'])
def test_resunet_inlier_forward_6d(abi, path):
  from deepglobalregistration_b200.model import load_model
  sd = syn.resunet_state_dict(5, 1, 1, 3, 6)
  g = np.random.default_rng(0)
  c0 = _small_pair_cloud(1, 6000)
  n = len(c0)
  # correspondences: 40% consistent shifts (cluster in 6-D), the rest random
  c1 = c0[:, 1:] + np.array([3, -2, 1])
  rnd = g.random(n) < 0.6
  c1[rnd] = c0[g.integers(0, n, int(rnd.sum())), 1:]
  coords6 = np.concatenate([c0, c1], 1).astype(np.int32)
  want = orn.resunet_forward(sd, coords6, torch.ones(n, 1), 3, False)
  model = load_model('ResUNetBN2C')(1, 1, bn_momentum=0.05, conv1_kernel_size=3, normalize_feature=False, D=6)
  model.load_state_dict(sd)
  model = model.cuda().eval()
  got = _forward(model, coords6, path)
  _close(got, want, tol=5e-5, what='inlier logits')
