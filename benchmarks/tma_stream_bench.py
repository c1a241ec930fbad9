"""HBM -> SMEM streaming micro-benchmark (TMA box shapes / bulk copies / LDG). Prints GB/s."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gllm_b200.ops import lib as _lib  # noqa: E402

L = _lib.load()
rows, cols = 24576, 4096  # 201 MB, like the gate/up weight
w = torch.randn(rows, cols, device="cuda").bfloat16()
sink = torch.zeros(1, dtype=torch.int64, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def run(mode, box_rows, chunk, stages, cps, label):
    st = torch.cuda.current_stream().cuda_stream
    ts = []
    for i in range(6):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        rc = L.gllm_bench_tma_stream(w.data_ptr(), rows, cols, cols, mode, box_rows, chunk, stages, cps,
                                     sink.data_ptr(), st)
        assert rc == 0
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ms = sorted(ts[1:])[len(ts[1:]) // 2]
    print(f"{label:58s} {ms*1e3:8.1f} us  {rows*cols*2/ms/1e6:8.1f} GB/s", flush=True)


for cps in (1, 2, 4):
    for box in (32, 64, 128, 256):
        for stages in (4, 8):
            if stages * box * 128 * cps > 200 * 1024:
                continue
            run(0, box, 0, stages, cps, f"TMA 2D box 64x{box} strided, stages={stages}, CTAs/SM={cps}")
for cps in (1, 2, 4):
    for chunk in (4096, 8192, 16384, 32768):
        for stages in (4, 8):
            if stages * chunk * cps > 200 * 1024:
                continue
            run(1, 0, chunk, stages, cps, f"bulk 1D {chunk} B contiguous, stages={stages}, CTAs/SM={cps}")
for cps in (2, 4, 8):
    run(2, 0, 16384, 1, cps, f"LDG.128 512 thr, CTAs/SM={cps}")
