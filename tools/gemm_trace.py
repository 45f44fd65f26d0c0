"""Per-tile timeline (SM clock cycles) of CTA 0 of the tensor-core GEMM for one short-K shape."""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from animate3d_b200 import _lib as L
from tools import kernel_bench as kb

lib = L.load()
buf = torch.zeros(1024, dtype=torch.int64, device="cuda")
which = sys.argv[1] if len(sys.argv) > 1 else "qkv"
lib.a3d_debug_set_gemm_trace(C.c_void_p(buf.data_ptr()))
M0 = 131072
if which == "qkv":
    kb.gemm_case("l0 qkv 320->1536 (traced)", M0, 1536, 320)
elif which == "geglu":
    kb.gemm_case("l0 geglu 320->2560 (traced)", M0, 2560, 320, geglu=True)
elif which == "sqkv":
    kb.gemm_case("l0 sqkv+rowbias (traced)", M0, 1152, 320, rowbias=True)
else:
    kb.gemm_case("l0 proj+res (traced)", M0, 320, 320, res=True)
lib.a3d_debug_set_gemm_trace(C.c_void_p(None))
t = buf.cpu().view(64, 16)
t0 = int(t[0, 0])
names = {0: "tile_start", 1: "mainloop_done", 2: "epilogue_done"}
order = [0, 1, 2]
print("tile " + " ".join(f"{names[k]:>13s}" for k in order))
for j in list(range(0, 14)) + [30, 31, 32]:
    print(f"{j:4d} " + " ".join(f"{int(t[j, k]) - t0:13d}" for k in order))
