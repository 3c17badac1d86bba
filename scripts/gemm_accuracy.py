"""Accuracy of the dense-layer kernels against an fp64 matmul: max |err| / max |y| and rms(err) / rms(y) for the wgmma
split-fp16 kernel, the FFMA kernel and torch's fp32 matmul (cuBLAS, allow_tf32 off), over several reduction lengths."""
import os, sys
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from nflows_b200 import kernels as K
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda:0")
def report(name, y, ref):
    e = (y.double() - ref)
    print("   %-14s max %.2e   rms %.2e" % (name, float(e.abs().max() / ref.abs().max()), float(e.pow(2).mean().sqrt() / ref.pow(2).mean().sqrt())))
for n, k, o, relu in ((4096, 16, 64, False), (4096, 24, 24, False), (4096, 256, 256, True), (4096, 784, 784, False), (4096, 256, 9408, True)):
    g = torch.Generator(device=dev).manual_seed(k + o)
    x = torch.randn(n, k, device=dev, generator=g)
    if relu: x = x.clamp_min(0)
    w = torch.randn(o, k, device=dev, generator=g) / k ** 0.5
    ref = x.double() @ w.double().t()
    print("n=%d K=%d N=%d%s" % (n, k, o, " relu(x)" if relu else ""))
    for e in (6, 2):
        report("f16x3 exp=%d" % e, K.linear_f16x3(K.split_f16(x, e), K.split_f16(w, K.weight_exp(w)))[0], ref)
    report("ffma", K.linear(x, w), ref)
    report("torch fp32", x @ w.t(), ref)
