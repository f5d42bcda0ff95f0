"""persistent LSTM layer kernels alone: fwd / bwd ms at the prediction-net shape (B=32, U+1=151, H=1024), one direction"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pika_b200 import kernels as K
B, U, H = int(os.environ.get("B", 32)), 151, 1024
g = torch.Generator(device="cuda").manual_seed(1)
gx = (torch.randn(B, U, 4 * H, generator=g, device="cuda") * 0.5).unsqueeze(0)      # leading n_dir = 1 axis
whh = (torch.randn(4 * H, H, generator=g, device="cuda") * 0.03).bfloat16()
out = torch.empty(B, U, H, device="cuda", dtype=torch.bfloat16)
gates = torch.empty(1, U, B, 4 * H, device="cuda")
cs = torch.empty(1, U, B, H, device="cuda")
dout = (torch.randn(B, U, H, generator=g, device="cuda") * 0.1).bfloat16()
dG = torch.empty(1, U, B, 4 * H, device="cuda", dtype=torch.bfloat16)
def t(fn, it=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(it): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / it
f = t(lambda: K.lstm_seq_fwd_ex(gx, whh, out, gates, cs))
b = t(lambda: K.lstm_seq_bwd_ex(dout, gates, cs, whh, dG))
print("fwd %.3f ms (%.2f us/step)  bwd %.3f ms (%.2f us/step)  checksum %.4f %.4f" %
      (f, f * 1e3 / U, b, b * 1e3 / U, out.float().abs().mean().item(), dG.float().abs().mean().item()))
