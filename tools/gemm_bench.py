"""Timing of the wgmma GEMM entry (egnn_gemm_bf16) over a few shapes: separates per-tile fixed cost from per-k cost."""
import os, sys, torch
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO]
from egnn_pytorch_b200 import _native as nat
lib = nat.load()
WAVE = 2 * torch.cuda.get_device_properties(0).multi_processor_count      # tiles in flight: two CTAs per SM
def t(M, N, K, out_f32=1, iters=20):
    A = torch.randn(M, K, device="cuda").bfloat16(); W = torch.randn(N, K, device="cuda").bfloat16()
    o = torch.empty(M, N, device="cuda", dtype=torch.float32 if out_f32 else torch.bfloat16)
    for _ in range(3): lib.egnn_gemm_bf16(M, N, K, A.data_ptr(), W.data_ptr(), None, 1.0, 0, o.data_ptr(), out_f32, None)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters): lib.egnn_gemm_bf16(M, N, K, A.data_ptr(), W.data_ptr(), None, 1.0, 0, o.data_ptr(), out_f32, None)
    b.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    tiles = ((M + 127) // 128) * ((N + 127) // 128)
    print(f"M={M:6d} N={N:5d} K={K:5d} f32out={out_f32}: {ms*1e3:8.1f} us  {2*M*N*K/ms/1e9:7.1f} TFLOP/s  tiles={tiles}  us/tile-wave={ms*1e3/max(1,(tiles+WAVE-1)//WAVE):.1f}")
for shape in [(128, 128, 512), (128, 128, 4096), (4096, 2112, 512), (4096, 2112, 64), (4096, 2112, 4096), (8192, 8192, 8192), (4096, 1024, 528), (4096, 512, 1024), (32768, 1088, 256)]:
    t(*shape)
t(4096, 2112, 512, out_f32=0)
