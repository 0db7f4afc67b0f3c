"""Per-phase cycle counters of the cluster GRU kernels (CTA 0 of each launch) over one eager C2 training step
(batch 256): encoder forward, decoder forward, decoder BPTT, encoder BPTT.  Cycles per time step.
Usage: python scripts/gru_phases.py [split]"""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import mtad_gat_pytorch_b200 as mg
from mtad_gat_pytorch_b200._lib import lib

SLOTS = 4                    # the step's four recurrence launches, in launch order
PHASES = ["mma.wait_operand", "mma.issue", "mma.wait_mma", "mma.store", "epi.wait_acc", "epi.math", "epi.send", "epi.tail"]
NAMES = {0: ["encoder fwd", "decoder fwd"], 1: ["decoder bptt", "encoder bptt"]}

torch.manual_seed(0)
m = mg.MTAD_GAT(38, 100, 38, forecast_n_layers=3, dropout=0.3).cuda().train()
m.branch_parallel = False
x = torch.rand(256, 100, 38, device="cuda")
y = torch.rand(256, 38, device="cuda")
if len(sys.argv) > 1:
    mg.set_gru_split(int(sys.argv[1]))
dbg = torch.zeros(SLOTS, 16, dtype=torch.int64, device="cuda")
for trial in range(2):                         # the first pass also loads the modules
    dbg.zero_()
    lib.mtadgat_gru_debug_buffer(dbg.data_ptr(), SLOTS)
    p, r = m(x)
    loss = torch.sqrt(torch.mean((p - y) ** 2)) + torch.sqrt(torch.mean((r - x) ** 2))
    loss.backward()
    torch.cuda.synchronize()
    lib.mtadgat_gru_debug_buffer(None, 0)
    m.zero_grad(set_to_none=True)
v = dbg.cpu().tolist()
seen = {0: 0, 1: 0}
print("launch".ljust(14) + "".join(p.rjust(17) for p in PHASES) + "   mma sum   epi sum  steps")
for row in v:
    if row[8] == 0:
        continue
    kind = row[9]
    name = NAMES[kind][min(seen[kind], 1)]
    seen[kind] += 1
    print(name.ljust(14) + "".join(str(c).rjust(17) for c in row[:8]) +
          str(sum(row[0:4])).rjust(10) + str(sum(row[4:8])).rjust(10) + str(row[8]).rjust(7))
