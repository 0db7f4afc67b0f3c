"""GAT layers forward (eval + train) at SMD shape, B=256, for ncu captures of the projection GEMM and score kernel."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mtad_gat_pytorch_b200 as mg
torch.manual_seed(0)
m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3).cuda()
x = torch.rand(256, 100, 38, device="cuda")
for it in range(3):
    m.eval()
    with torch.no_grad():
        m.feature_gat(x); m.temporal_gat(x)
    m.train()
    xi = x.clone().requires_grad_(True)
    m.feature_gat(xi); m.temporal_gat(xi)
torch.cuda.synchronize()
print("done")
