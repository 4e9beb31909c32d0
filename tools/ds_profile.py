import sys, os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "moe-infinity_b200")); sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch, bench_configs as B
from moe_infinity_b200 import MoEEngine, _lib as L
Hh, I, E, k, Lr, T = 2048, 1408, 64, 6, 4, int(os.environ.get("DS_T", "16"))
eng = MoEEngine(num_layers=Lr, num_experts=E, hidden=Hh, inter=I, top_k=k, dtype=torch.bfloat16, expert_type=L.EXPERT_DEEPSEEK,
                router=L.ROUTER_DEEPSEEK_GREEDY, shared_inter=2 * I, max_tokens=T, num_slots=Lr * E)
for l in range(Lr):
    for e in range(E):
        eng.load_expert(l, e).normal_(0, 0.02)
    eng.set_gate(l, torch.randn(E, Hh, device="cuda") * 0.05)
    eng._ck(eng.lib.b2m_register_shared(eng._h, l, None, 0))
x = torch.randn(Lr, T, Hh, device="cuda").to(torch.bfloat16)
out = torch.empty_like(x)
for it in range(3):
    for l in range(Lr):
        eng.forward(l, x[l], out=out[l])
torch.cuda.synchronize()
