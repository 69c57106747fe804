"""ME.utils: sparse_quantize / batched_coordinates as called at
core/deep_global_registration.py:152,158 (ME 0.5 return convention)."""
import numpy as np
import torch

from .. import _abi


def sparse_quantize(coordinates, features=None, labels=None, ignore_label=-100, return_index=False,
                    return_inverse=False, return_maps_only=False, quantization_size=None, device='cuda'):
  """Floor the (already scaled) coordinates and keep the first point of every voxel.
  Returns unique integer coordinates [+ features] [+ index] [+ inverse] in first-occurrence
  order; `index` are ascending rows of the input.  The work runs on the GPU; results come
  back in the container type of the input (numpy in -> numpy out)."""
  if labels is not None:
    raise NotImplementedError('label-aware quantisation is not on the DGR hot path')
  is_np = isinstance(coordinates, np.ndarray)
  c = torch.from_numpy(np.ascontiguousarray(coordinates)) if is_np else coordinates
  if quantization_size is not None:
    c = c / quantization_size
  dev = _abi.require_device(device if not c.is_cuda else c.device)
  c = c.to(dev)
  if c.shape[1] != 3:
    raise NotImplementedError('sparse_quantize is built for 3-D point clouds')
  if not c.dtype.is_floating_point:
    c = c.double()
  if c.dtype not in (torch.float32, torch.float64):
    c = c.float()
  coords, _, _, sel, inverse, _ = _abi.voxelise(c.contiguous(), 1.0)
  index = sel.long()
  uniq = coords[index][:, 1:].contiguous()
  conv = (lambda t: t.cpu().numpy()) if is_np else (lambda t: t)
  if return_maps_only:
    return (conv(index), conv(inverse.long())) if return_inverse else conv(index)
  out = [conv(uniq)]
  if features is not None:
    f = features[index.cpu().numpy()] if isinstance(features, np.ndarray) else features[index.to(features.device)]
    out.append(f)
  if return_index:
    out.append(conv(index))
  if return_inverse:
    out.append(conv(inverse.long()))
  return out[0] if len(out) == 1 else tuple(out)


def batched_coordinates(coords, dtype=torch.int32, device=None):
  """[(N_b, D)] -> [sum N_b, D + 1] with the batch index in column 0."""
  out = []
  for b, c in enumerate(coords):
    if isinstance(c, np.ndarray):
      c = torch.from_numpy(c)
    c = c.to(dtype)
    out.append(torch.cat([torch.full((len(c), 1), b, dtype=dtype, device=c.device), c], 1))
  out = torch.cat(out, 0)
  return out.to(device) if device is not None else out


def kaiming_normal_(*a, **k):
  raise NotImplementedError('weight initialisers for training are outside the built hot path')
