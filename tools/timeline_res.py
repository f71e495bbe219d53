"""Debug helper: per-CTA timelines of the resident forward / backward kernels (TCR_DEBUG_TIMELINE=1): median time of each stamp
relative to the earliest CTA start of that kernel, and min / max over CTAs.
forward slots: 0 start; per phase ph<3 at 1+8ph: +0 bank ready, +1 fma done, +2 stats done (arrive), +3 y stored, +4 barrier passed,
+5 tables built, +6 next tile staged; 31 end.   backward slots: 0 start; per phase (Bb2,Ba2,Bb1,Ba1,Bb0,Ba0) at 1+5i: +0 inputs landed,
+1 convT done, +2 epilogue done (arrive), +3 prefetch issued, +4 barrier passed; 31 end."""
import os, sys, ctypes as C
import numpy as np, torch
os.environ["TCR_DEBUG_TIMELINE"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import tcresnet_b200  # noqa
from tcresnet_b200.engine import Engine
from tcresnet_b200 import _lib as L
N = int(sys.argv[1]) if len(sys.argv) > 1 else 512
eng = Engine(max_batch=N)
dev = eng.device
p, s, m = eng.new_variables(0)
wav = torch.rand(N, 16000, device=dev) * 2 - 1
hot = torch.nn.functional.one_hot(torch.randint(0, 12, (N,), device=dev), 12).float()
for i in range(5):
    eng.train_step(wav, hot, p, s, m, 0.1)
torch.cuda.synchronize()
ptr, numel = C.c_void_p(), C.c_int64()
L.check(eng.lib, eng.lib.tcr_workspace_tensor(eng._h, b"timeline", C.byref(ptr), C.byref(numel)), "timeline")
buf = torch.empty(2 * 148 * 32, dtype=torch.int64, device=dev)
rt = C.CDLL('libcudart.so.12')
rt.cudaMemcpy.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
assert rt.cudaMemcpy(buf.data_ptr(), ptr.value, 2 * 148 * 32 * 8, 3) == 0
tt = buf.cpu().numpy().reshape(2, 148, 32).astype(np.float64)
for name, t in zip(("forward", "backward"), tt):
    if not (t[:, 0] > 0).any():
        continue
    t0 = t[:, 0][t[:, 0] > 0].min()
    print(name)
    prev = 0.0
    for sl in range(32):
        col = t[:, sl]
        col = col[col > 0]
        if not len(col):
            continue
        med = np.median(col) - t0
        print(f"  {sl:2d} median {med/1e3:8.2f} us  (+{(med-prev)/1e3:6.2f})  min {(col.min()-t0)/1e3:8.2f}  max {(col.max()-t0)/1e3:8.2f}")
        prev = med
