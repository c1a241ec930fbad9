"""Fused TP vs NCCL baseline micro-benchmark for one decoder block's communication pattern (run under torchrun).
Times (CUDA events, max over ranks) per T:  O-proj[+reduce]+add+norm -> gate/up GEMM -> down[+reduce]+add+norm -> QKV GEMM
    torchrun --nproc-per-node N benchmarks/tp_bench.py
"""
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    from gllm_b200.parallel import state as ps
    ps.init_dist(1, world, rank, local)
    from gllm_b200.ops import ref, sm100
    from gllm_b200.parallel.fused import FusedTPComm
    from gllm_b200.parallel.tp import TPComm
    dev = torch.device("cuda", local)
    H, I, QKV, HQ = 4096, 12288 // world, 6144 // world, 4096 // world
    torch.manual_seed(rank)
    w_o = (torch.randn(H, HQ, device=dev) * 0.02).bfloat16()
    w_gu = ref.interleave_gate_up((torch.randn(2 * I, H, device=dev) * 0.02).bfloat16(), 128)
    w_dn = (torch.randn(H, I, device=dev) * 0.02).bfloat16()
    w_qkv = (torch.randn(QKV, H, device=dev) * 0.02).bfloat16()
    nw = torch.ones(H, device=dev).bfloat16()
    fused = FusedTPComm(max_tokens=8192, hidden_size=H, device=dev)
    base = TPComm(sm100)

    def block(tpc, a, res):
        h, res = tpc.row_linear_add_norm(a, w_o, res, nw, 1e-6)
        act = tpc.col_linear_silu_mul(h, w_gu)
        h, res = tpc.row_linear_add_norm(act, w_dn, res, nw, 1e-6)
        return tpc.col_linear(h, w_qkv), res

    for T in (32, 256, 1024, 4096):
        a = (torch.randn(T, HQ, device=dev) * 0.5).bfloat16()
        x0 = (torch.randn(T, H, device=dev) * 0.5).bfloat16()
        out = {}
        for name, tpc in (("nccl", base), ("fused", fused)):
            def run():
                tpc.begin_forward(T)
                h, res = tpc.first_norm(x0, nw, 1e-6)
                if name == "nccl":
                    res = res.clone()
                y = None
                for _ in range(4):  # 4 blocks per measurement (even number of RS calls)
                    y, res = block(tpc, a, res)
                return y
            for _ in range(5):
                run()
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            iters = 20
            e0.record()
            for _ in range(iters):
                run()
            e1.record()
            torch.cuda.synchronize()
            t = torch.tensor([e0.elapsed_time(e1) / iters / 4], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            out[name] = round(t.item() * 1e3, 1)
            dist.barrier()
        if rank == 0:
            print(json.dumps({"tp": world, "T": T, "us_per_block_nccl": out["nccl"], "us_per_block_fused": out["fused"],
                              "speedup": round(out["nccl"] / out["fused"], 3)}), flush=True)
    dist.barrier()
    sys.stdout.flush()
    os._exit(0)


if __name__ == "__main__":
    main()
