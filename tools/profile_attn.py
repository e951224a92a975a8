"""Time the two attention kernels on one shape (for ncu / A-B):  python tools/profile_attn.py B L [tc_mode] [reps]
Prints per-launch microseconds of the tensor-core kernel (attention_tc.cu) and the fp32 FFMA flash kernel (am_kernels.cu)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from emotivoice_b200 import _abi, build

build.build(verbose=False)
lib = _abi.load()
B, L = int(sys.argv[1]), int(sys.argv[2])
tc_mode = int(sys.argv[3]) if len(sys.argv) > 3 else 1
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 5
H, heads = 384, 8
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(1)
qkv = torch.randn(B, L, 3 * H, generator=g).to(dev)
out = torch.empty(B, L, H, device=dev)
flush = torch.empty(64 * 1024 * 1024, device=dev)
st = torch.cuda.current_stream().cuda_stream
res = {}
for name, fn in (("tc", lambda: lib.ev_op_attention_tc(qkv.data_ptr(), None, out.data_ptr(), B, L, H, heads, tc_mode, st)),
                 ("ffma", lambda: lib.ev_op_attention(qkv.data_ptr(), None, out.data_ptr(), B, L, H, heads, st))):
    ts = []
    for i in range(reps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        _abi.check(fn())
        e1.record()
        e1.synchronize()
        ts.append(round(e0.elapsed_time(e1) * 1e3, 1))
    res[name] = ts
flop = 4.0 * B * heads * L * L * 48
print(json.dumps({"B": B, "L": L, "tc_mode": tc_mode, "us": res, "tflops_tc": round(flop / min(res["tc"][1:]) / 1e6, 1),
                  "tflops_ffma": round(flop / min(res["ffma"][1:]) / 1e6, 1)}))
