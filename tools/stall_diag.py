"""Where do the periodic slow steps of register() come from?  300 steps on one pair, host-side
wall time per phase (synchronising after each phase), allocator statistics before / after."""
import gc, os, sys, time, types
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from deepglobalregistration_b200 import _abi, synthetic as syn
from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration

state = syn.make_checkpoint(0)
dgr = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False))
dgr.use_icp = False
pairs = [syn.room_pair(i, n_raw=250000) for i in range(3)]
pdev = [(torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()) for a, b, _ in pairs]
mode = sys.argv[1] if len(sys.argv) > 1 else 'phases'
for i in range(12): dgr.register(*pdev[i % 3])
torch.cuda.synchronize(); gc.collect(); gc.disable()
st0 = torch.cuda.memory_stats()
def sync(): torch.cuda.synchronize(); return time.perf_counter()
rows = []
t_begin = time.perf_counter()
for step in range(300):
  a, b = pdev[step % 3]
  t = [sync()]
  if mode == 'plain':
    dgr.register(a, b); t.append(sync())
  else:
    with torch.no_grad():
      _abi.refresh_stream()
      x0, c0, _ = dgr.preprocess(a, 0, _batch=0); x1, c1, _ = dgr.preprocess(b, 1, _batch=1); t.append(sync())
      F0, F1 = dgr.fcgf_feature_extraction_pair(c0, c1); t.append(sync())
      idx1 = _abi.knn_top1(F0, F1); t.append(sync())
      c6 = _abi.inlier_coords(c0, c1, idx1)
      logit = dgr._stage_forward(dgr.native_networks()[1], c6, unique=True); t.append(sync())
      w, ws = _abi.sigmoid_clip_sum(logit, 0.05)
      res = _abi.se3_register(x0, x1, w.reshape(-1), idx1=idx1, quantization_size=0.1, break_threshold_ratio=1e-4).cpu(); t.append(sync())
  rows.append((t[0] - t_begin, [1e3 * (y - x) for x, y in zip(t[:-1], t[1:])]))
st1 = torch.cuda.memory_stats()
tot = np.array([sum(r[1]) for r in rows])
print(mode, 'median %.2f mean %.2f max %.1f  n>25ms %d' % (np.median(tot), tot.mean(), tot.max(), (tot > 25).sum()))
for k in ('num_device_alloc', 'num_device_free', 'num_alloc_retries', 'reserved_bytes.all.current', 'num_sync_all_streams'):
  print(' ', k, st0.get(k), '->', st1.get(k))
names = ['preproc', 'fcgf', 'knn', 'inlier', 'refine+read']
med = np.median(np.array([r[1] for r in rows]), 0) if mode != 'plain' else None
if med is not None: print('  median per phase', dict(zip(names, np.round(med, 2))))
for ts, ph in rows:
  if sum(ph) > 25: print('  t=%.2fs total %.1f' % (ts, sum(ph)), dict(zip(names, np.round(ph, 1))) if mode != 'plain' else '')
