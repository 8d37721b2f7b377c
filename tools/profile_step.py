"""Warm, in-pipeline per-kernel GPU times of one GPSLayer fwd+bwd step (torch.profiler / CUPTI)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import graphgps_b200
from graphgps_b200.graph import graph_of
from torch.profiler import profile, ProfilerActivity

wl = sys.argv[1] if len(sys.argv) > 1 else "pcqm4m-small"
precision = sys.argv[2] if len(sys.argv) > 2 else "fp32"
local, glob, heads, drop, adrop = {"pcqm4m-small": ("CustomGatedGCN", "Transformer", 4, 0.0, 0.5),
                                   "pcqm4m-medium-performer": ("CustomGatedGCN", "Performer", 16, 0.1, 0.1),
                                   "zinc-gine": ("GINE", "Transformer", 4, 0.0, 0.5),
                                   "code2": ("CustomGatedGCN", "Transformer", 4, 0.2, 0.2)}[wl]
spec = graphgps_b200.SHAPES[wl]
dev = "cuda:0"
torch.manual_seed(0)
layer = graphgps_b200.GPSLayer(spec.dim, local, glob, heads, dropout=drop, attn_dropout=adrop,
                              precision=precision).to(dev).train()
b = graphgps_b200.make_batch(wl, seed=0).to(dev)
graph_of(b)
ct_x, ct_e = torch.randn_like(b.x), torch.randn_like(b.edge_attr)

def step():
    bb = graphgps_b200.GraphBatch(x=b.x.detach().requires_grad_(True), edge_index=b.edge_index,
                                  edge_attr=b.edge_attr.detach().requires_grad_(True), batch=b.batch, num_graphs=b.num_graphs)
    bb.__dict__["_gps_b200_graph"] = b.__dict__["_gps_b200_graph"]
    for p in layer.parameters():
        p.grad = None
    out = layer(bb)
    if local == "CustomGatedGCN":
        torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
    else:
        torch.autograd.backward([out.x], [ct_x])

for _ in range(5):
    step()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(10):
        step()
    torch.cuda.synchronize()
rows = []
for e in prof.key_averages():
    if e.device_type is not None and getattr(e, "device_time_total", 0) > 0:
        rows.append((e.device_time_total / 10.0, e.count / 10.0, e.key))
rows.sort(reverse=True)
tot = sum(r[0] for r in rows)
print(f"{wl} {precision}: sum of kernel time per step = {tot:.1f} us")
for t, c, k in rows[:28]:
    k = k.replace("gps::(anonymous namespace)::", "").replace("void ", "")
    print(f"{t:9.1f} us {100*t/tot:5.1f}%  n={c:4.1f}  avg={t/c:7.1f}  {k[:90]}")

# ---- timeline of ONE step: (start offset us, duration us, stream, kernel) to see the critical path / overlap
with profile(activities=[ProfilerActivity.CUDA]) as prof2:
    step()
    torch.cuda.synchronize()
evs = [e for e in prof2.events() if e.device_type is not None and str(e.device_type).endswith("CUDA") and e.time_range is not None]
evs = [e for e in evs if (e.time_range.end - e.time_range.start) > 0]
evs.sort(key=lambda e: e.time_range.start)
if evs:
    t0 = evs[0].time_range.start
    print("timeline of one step: start_us dur_us stream name")
    for e in evs:
        nm = e.name.replace("gps::(anonymous namespace)::", "").replace("void ", "")[:60]
        print(f"{e.time_range.start - t0:8.1f} {e.time_range.end - e.time_range.start:7.1f}  s{getattr(e, 'stream', getattr(e, 'device_resource_id', '?'))}  {nm}")
    print("step span us:", evs[-1].time_range.end - t0)
