"""Small profiling target (development tool): a few launches of each hot kernel on a 64k batch, for
   ncu --set full -k regex:<kernel> -s <skip> -c 1 python tools/ncu_target.py
   Each keyed call below is two kernels: ecdsa_prep_kernel (the scalars), then ecdsa_verify_cached_kernel (the chain)."""
import importlib, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("fabric-mod_b200")
from tools import workload
n = 65536
w = workload.Workload(n, 64, seed=workload.DEFAULT_SEED + 2)
ctx = pkg.binding.Context(max_batch=n)
dev = torch.device("cuda:0")
t = [torch.from_numpy(a).to(dev) for a in (w.qx(), w.qy(), w.digest, w.r, w.s)]
slots = ctx.keys_register(w.keys_xy) & 0xFFF          # device-resident API takes raw slot indices
ks = torch.from_numpy(slots[w.key_idx]).to(dev)
mask = torch.zeros(n // 32, dtype=torch.int32, device=dev)
st = torch.cuda.current_stream(dev)
for _ in range(4):
    ctx.verify_p256_device_keyed(True, ks.data_ptr(), 0, 0, t[2].data_ptr(), t[3].data_ptr(), t[4].data_ptr(), n, mask.data_ptr(), 0, st.cuda_stream)
torch.cuda.synchronize()
assert bool((mask == -1).all())
for _ in range(2):
    ctx.verify_p256_device(*[x.data_ptr() for x in t], n, mask.data_ptr(), 0, st.cuda_stream)
torch.cuda.synchronize()
assert bool((mask == -1).all())
# SHA-256: 60k messages shaped like a block's (payload-sized and endorsement-sized)
rng = np.random.default_rng(1)
buf = rng.integers(0, 256, 64 << 20, dtype=np.uint8)
jobs = np.zeros((60000, 6), np.uint32)
jobs[:, 0] = rng.integers(0, (64 << 20) - 8192, 60000)
jobs[:10000, 3] = 4300
jobs[10000:40000, 3] = 330
jobs[10000:40000, 1] = rng.integers(0, (64 << 20) - 8192, 30000)
jobs[10000:40000, 4] = 1100
jobs[40000:, 3] = 1200
for _ in range(2):
    d = ctx.sha256_segments(buf, jobs)
print("ncu target done")
