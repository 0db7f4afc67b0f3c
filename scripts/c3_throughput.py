"""Forward-only scoring throughput at the C3 config (MSL shape k=55, n=100, out=1, batch 4096)."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mtad_gat_pytorch_b200 as mg
torch.manual_seed(0)
m = mg.MTAD_GAT(55, 100, 1, forecast_n_layers=3, dropout=0.3).cuda().eval()
x = torch.rand(4096, 100, 55, device="cuda")
flush = torch.empty(256 * 1024 * 1024 // 4, device="cuda")
with torch.no_grad():
    for _ in range(3):
        m(x)
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream(); s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m(x)
    torch.cuda.current_stream().wait_stream(s); torch.cuda.synchronize()
    with torch.cuda.graph(g, stream=s):
        out = m(x)
    ts = []
    for _ in range(10):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); g.replay(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
ts.sort()
print(json.dumps({"config": "C3 MSL-shape forward, batch 4096", "ms": ts[len(ts) // 2], "windows_per_s": 4096 / (ts[len(ts) // 2] * 1e-3)}))
