"""Times the captured training-step CUDA graph of the medical CNN (tcgen05 engine): median of
N replays on fresh data indices, L2 flushed between replays."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from hefl_b200.config import FLConfig
from hefl_b200.models import ParamPack, create_model
from hefl_b200.fl.trainer import LocalTrainer

cfg = FLConfig(model="medcnn", batch_size=32, nn_backend="tcgen05")
dev = torch.device("cuda")
model = create_model("medcnn").to(dev)
pack = ParamPack(model)
tr = LocalTrainer(model, pack, cfg, dev, backend="tcgen05", use_graph=True)
x = torch.randint(0, 256, (32, 256, 256, 3), dtype=torch.uint8, device="cuda")
y = torch.randint(0, 2, (32,), device="cuda")
for _ in range(5):
    tr.train_step(x, y)
torch.cuda.synchronize()
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
ts = []
for _ in range(20):
    flush.zero_()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record(); tr.train_step(x, y); e.record(); torch.cuda.synchronize()
    ts.append(s.elapsed_time(e) * 1e3)
ts.sort()
# back-to-back replays (what a round does)
s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
s.record()
for _ in range(50):
    tr.train_step(x, y)
e.record(); torch.cuda.synchronize()
print(f"graph step median {ts[len(ts)//2]:.1f} us (L2 flushed), back-to-back {s.elapsed_time(e)*1e3/50:.1f} us/step, loss {tr.out_train.tolist()}")
