"""Warm, in-pipeline per-kernel GPU times of one GPSLayer fwd+bwd step (torch.profiler / CUPTI).

    python tools/profile_step.py [workload] [fp32|bf16]

Prints the per-kernel totals of ten steps, then one step's timeline per direction (start offset, duration, stream,
kernel) and a branch summary: the layer step is a trunk that forks into the local-model branch (on the caller's
stream) and the global-attention branch (on its own stream) and joins before norm1 in the forward and before the g_x
product in the backward.  Only the longer branch of each pair is on the critical path."""
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


def forward():
    bb = graphgps_b200.GraphBatch(x=b.x.detach().requires_grad_(True), edge_index=b.edge_index,
                                  edge_attr=b.edge_attr.detach().requires_grad_(True), batch=b.batch, num_graphs=b.num_graphs)
    bb.__dict__["_gps_b200_graph"] = b.__dict__["_gps_b200_graph"]
    for p in layer.parameters():
        p.grad = None
    return layer(bb)


def backward(out):
    if local == "CustomGatedGCN":
        torch.autograd.backward([out.x, out.edge_attr], [ct_x, ct_e])
    else:
        torch.autograd.backward([out.x], [ct_x])


def step():
    backward(forward())


def short(name):
    return name.replace("gps::(anonymous namespace)::", "").replace("void ", "")


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
    print(f"{t:9.1f} us {100*t/tot:5.1f}%  n={c:4.1f}  avg={t/c:7.1f}  {short(k)[:90]}")


def timeline(fn):
    """GPU activities of fn() as (start us, end us, stream, name), sorted by start; fn ends in a synchronise."""
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        res = fn()
        torch.cuda.synchronize()
    evs = [e for e in p.events() if e.device_type is not None and str(e.device_type).endswith("CUDA")
           and e.time_range is not None and e.time_range.end > e.time_range.start]
    evs = [(e.time_range.start, e.time_range.end, getattr(e, "device_resource_id", "?"), short(e.name)) for e in evs]
    evs.sort()
    return evs, res


def is_attention(name):
    return "k_attn" in name or "k_perf" in name


def branch_summary(direction, evs, main):
    """Spans of the trunk before the fork, both branches and the trunk after the join, from one direction's timeline.
    The attention branch is every activity on the stream that runs the attention kernels; its first activity marks
    the fork.  The join is the first main-stream kernel that waits for both branches: norm1's bn_combine in the
    forward, the g_x product (the last main-stream kernel) in the backward.  The local branch is the main stream's
    work between the fork and the join."""
    evs = [e for e in evs if not e[3].startswith("at::")]   # torch's own kernels ahead of the layer's work
    t0, t_end = evs[0][0], max(e[1] for e in evs)
    attn_streams = {e[2] for e in evs if is_attention(e[3])}
    if not attn_streams:
        print(f"{direction}: no attention branch")
        return
    sa = attn_streams.pop()
    on_a = [e for e in evs if e[2] == sa]
    fork = on_a[0][0]
    on_main = [e for e in evs if e[2] == main]
    if direction == "forward":
        join = next(e for e in on_main if "OpCombine" in e[3] and e[0] >= fork)
    else:
        join = on_main[-1]
    loc = [e for e in on_main if e[0] >= fork and e[1] <= join[0]]
    a_end = max(e[1] for e in on_a if e[1] <= join[0])
    l_end = max(e[1] for e in loc) if loc else fork
    l_span, a_span = l_end - fork, a_end - fork
    bound = "local" if l_span >= a_span else "attention"
    print(f"{direction}: trunk before fork {fork - t0:7.1f} us | local branch {l_span:7.1f} us busy "
          f"{sum(e[1] - e[0] for e in loc):7.1f} us | attention branch {a_span:7.1f} us busy "
          f"{sum(e[1] - e[0] for e in on_a if e[1] <= join[0]):7.1f} us | join wait {join[0] - max(l_end, a_end):5.1f} us"
          f" | trunk after join {t_end - join[0]:7.1f} us | span {t_end - t0:7.1f} us | bound by {bound} "
          f"(by {abs(l_span - a_span):.1f} us)")
    crit = loc if bound == "local" else [e for e in on_a if e[1] <= join[0]]
    top = max(crit, key=lambda e: e[1] - e[0]) if crit else None
    print(f"  join kernel: {join[3][:80]}")
    if top:
        print(f"  longest kernel on the bounding branch: {top[1] - top[0]:6.1f} us  {top[3][:80]}")


# ---- timeline of ONE step per direction (start offset us, duration us, stream, kernel) and its branch summary
step()
torch.cuda.synchronize()
fwd_evs, out = timeline(forward)
bwd_evs, _ = timeline(lambda: backward(out))
main = fwd_evs[0][2]   # the forward's first launch (weight packing) is on the caller's stream
for direction, evs in (("forward", fwd_evs), ("backward", bwd_evs)):
    t0 = evs[0][0]
    print(f"timeline of one {direction} pass: start_us dur_us stream name")
    for s, e, sid, nm in evs:
        print(f"{s - t0:8.1f} {e - s:7.1f}  s{sid}  {nm[:60]}")
    print(f"{direction} span us:", max(e[1] for e in evs) - t0)
print(f"branch summary, {wl} {precision} (main stream s{main}):")
for direction, evs in (("forward", fwd_evs), ("backward", bwd_evs)):
    branch_summary(direction, evs, main)
