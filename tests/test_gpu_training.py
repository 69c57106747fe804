"""Training path (SURVEY 8f rank 3): backward of the sparse convolution and a training step through the ME-shaped
modules.  Parity by autograd through the oracle's plain-torch operators (oracle/sparse_ops.py): gradients are free
there.  Tolerances: fp32 gradients <= 2e-5 relative to the largest entry."""
import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import sparse_ops as so

pytestmark = pytest.mark.gpu


def _cloud(D, n, ext, seed):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-ext, ext, size=(n, D)), axis=0)
  c = c[g.permutation(len(c))]
  return np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)


@pytest.mark.parametrize('D,cin,cout,stride,transpose', [(3, 32, 64, 1, False), (3, 16, 24, 2, False), (3, 64, 32, 2, True),
                                                         (6, 8, 16, 1, False), (3, 1, 32, 1, False)])
def test_conv_backward_matches_oracle_autograd(D, cin, cout, stride, transpose):
  from deepglobalregistration_b200 import me as ME
  ME.set_conv_mode('tc3')
  coords = _cloud(D, 3000 if D == 3 else 2500, 9 if D == 3 else 3, seed=cin + cout)
  g = torch.Generator().manual_seed(cout)
  maps = so.CoordinateMaps(coords)
  if stride == 1:
    buckets, n_in, n_out = maps.same_map(1, 3), len(coords), len(coords)
  else:
    down = maps.down_map(1)
    n_fine, n_coarse = len(coords), len(maps.coords_at(2))
    buckets, n_in, n_out = (so.swap_map(down), n_coarse, n_fine) if transpose else (down, n_fine, n_coarse)
  K = 3 ** D
  x = torch.randn(n_in, cin, generator=g)
  w = torch.randn(K, cin, cout, generator=g) / np.sqrt(cin * 6)
  gout = torch.randn(n_out, cout, generator=g)
  # oracle: plain torch, autograd
  xo, wo = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
  (so.conv_forward(xo, wo, buckets, n_out) * gout).sum().backward()
  # CUDA path through the ME-shaped modules
  if transpose:
    conv = ME.MinkowskiConvolutionTranspose(cin, cout, kernel_size=3, stride=2, dimension=D).cuda().train()
    # a transposed convolution needs its matching strided convolution's map: run a 1-channel one first
    down_conv = ME.MinkowskiConvolution(1, cin, kernel_size=3, stride=2, dimension=D).cuda().train()
    st_fine = ME.SparseTensor(torch.ones(len(coords), 1), coordinates=torch.from_numpy(coords), device='cuda')
    coarse = down_conv(st_fine)
    xin = ME.SparseTensor(x.cuda().requires_grad_(True), coordinate_map_key=coarse.coordinate_map_key,
                          coordinate_manager=coarse.coordinate_manager)
  else:
    conv = ME.MinkowskiConvolution(cin, cout, kernel_size=3, stride=stride, dimension=D).cuda().train()
    xin = ME.SparseTensor(x.cuda().requires_grad_(True), coordinates=torch.from_numpy(coords), device='cuda')
  with torch.no_grad():
    conv.kernel.copy_(w.cuda())
  out = conv(xin)
  assert out.F.shape == (n_out, cout)
  (out.F * gout.cuda()).sum().backward()
  gx, gw = xin.F.grad.cpu(), conv.kernel.grad.cpu()

  def rel(a, b):
    return float((a - b).abs().max() / (1e-12 + b.abs().max()))
  assert rel(gx, xo.grad) <= 2e-5, rel(gx, xo.grad)
  assert rel(gw, wo.grad) <= 2e-5, rel(gw, wo.grad)


def test_training_step_then_native_inference():
  """ResUNetBN2C in train() mode (BatchNorm on batch statistics): loss.backward() reaches every parameter, the
  gradients are finite, running statistics move, and two SGD steps reduce the loss."""
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.model import load_model
  torch.manual_seed(0)
  net = load_model('ResUNetBN2C')(1, 16, bn_momentum=0.05, conv1_kernel_size=3, normalize_feature=False, D=3).cuda().train()
  coords = torch.from_numpy(_cloud(3, 4000, 10, seed=1))
  target = torch.randn(len(coords), 16, device='cuda')
  opt = torch.optim.SGD(net.parameters(), lr=1e-2)
  rm0 = net.norm1.bn.running_mean.clone()
  losses = []
  for _ in range(3):
    opt.zero_grad()
    out = net(ME.SparseTensor(torch.ones(len(coords), 1), coordinates=coords, device='cuda'))
    loss = ((out.F - target) ** 2).mean()
    loss.backward()
    losses.append(float(loss))
    for name, p in net.named_parameters():
      assert p.grad is not None and bool(torch.isfinite(p.grad).all()), name
    opt.step()
  assert losses[2] < losses[0], losses
  assert not torch.equal(rm0, net.norm1.bn.running_mean)
  # back to inference: eval() + no_grad() is the forward-only path and matches the native executor
  from deepglobalregistration_b200 import native
  net.eval()
  with torch.no_grad():
    x = ME.SparseTensor(torch.ones(len(coords), 1), coordinates=coords, device='cuda')
    a = net(x).F
  b = native.Net(net, 'cuda').forward(native.Context('cuda'), coords.cuda().contiguous(), x.F)
  assert float((a - b).abs().max()) <= 2e-5 * (1 + float(a.abs().max()))


def test_weighted_procrustes_backward_on_cuda():
  """The SVD backward of weighted_procrustes is torch's (the reference's own core/registration.py runs on torch
  ops); this checks the glue a training step needs: gradients flow from a pose loss through this package's
  Procrustes wrapper into the inlier logits."""
  from deepglobalregistration_b200.core import registration as reg
  X, tgt, _, idx1, T_gt, inl = syn.correspondence_set(2, n=800, inlier_frac=0.6)
  X, Y = torch.from_numpy(X).cuda(), torch.from_numpy(tgt[idx1]).cuda()
  logit = torch.zeros(len(X), 1, device='cuda', requires_grad=True)
  R, t = reg.weighted_procrustes_autograd(X, Y, torch.sigmoid(logit))
  loss = (R - torch.from_numpy(T_gt[:3, :3]).float().cuda()).pow(2).sum() + (t.reshape(-1) - torch.from_numpy(T_gt[:3, 3]).float().cuda()).pow(2).sum()
  loss.backward()
  assert bool(torch.isfinite(logit.grad).all()) and float(logit.grad.abs().max()) > 0
  # forward value equals the inference kernel's closed-form solution
  R_k, t_k = reg.weighted_procrustes(X, Y, torch.sigmoid(logit).detach())
  assert float((R.detach().cpu() - R_k).abs().max()) <= 5e-6 and float((t.detach().cpu() - t_k).abs().max()) <= 5e-6
