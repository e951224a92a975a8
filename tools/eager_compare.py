"""Secondary comparison (BASELINE.md s3 item 4): the reference's algorithm in EAGER PyTorch on the same H100
(cuDNN / cuBLAS library kernels; ~520 launches and 3 host syncs per utterance) next to the engine.
The oracle restatement issues exactly the torch ops the reference issues (it is bit-identical to it on CPU),
so running it on cuda:0 is the reference's own GPU path.  Test infrastructure, not product code."""
import json, os, statistics, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from emotivoice_b200 import synth
from emotivoice_b200.config import default_config
from emotivoice_b200.modules import JETSGenerator
from oracle import jets_oracle as O

dev = torch.device("cuda:0")
conf = default_config()
sd = synth.make_state_dict(conf)
sd_dev = {k: v.to(dev) for k, v in sd.items()}
batch = {k: v.to(dev) for k, v in synth.make_batch([100], seed=synth.SEED).items()}
res = {}
for tf32 in (False, True):
    torch.backends.cudnn.allow_tf32 = tf32
    torch.backends.cuda.matmul.allow_tf32 = False      # PyTorch defaults: conv TF32 on, matmul TF32 off
    for _ in range(3):
        o = O.jets_forward(sd_dev, conf, **batch)
    torch.cuda.synchronize()
    ts = []
    for _ in range(10):
        t0 = time.perf_counter(); o = O.jets_forward(sd_dev, conf, **batch); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    res["eager_cudnn_tf32_%s" % ("on(default)" if tf32 else "off")] = {"ms": 1e3 * statistics.median(ts), "frames": int(o["dec_outputs"].shape[1])}
m = JETSGenerator(conf).to(dev); m.load_state_dict(sd); m.eval()
for prec in ("fp32", "tf32"):
    m.precision = prec
    for _ in range(3):
        m(**batch)
    torch.cuda.synchronize()
    ts = []
    for _ in range(10):
        t0 = time.perf_counter(); m(**batch); torch.cuda.synchronize(); ts.append(time.perf_counter() - t0)
    res["engine_%s" % prec] = {"ms": 1e3 * statistics.median(ts)}
print(json.dumps(res))
