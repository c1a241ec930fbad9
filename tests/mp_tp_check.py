"""Multi-GPU check of the fused TP path (run under torchrun, one rank per GPU):
   1. op level : GEMM⊕reduce-scatter -> add+RMSNorm -> all-gather⊕GEMM  vs  NCCL all_reduce + torch math
   2. engine   : tokens of tp_mode=fused == tokens of tp_mode=nccl on a small random model
Prints 'TP_CHECK_OK' on rank 0 on success."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    import faulthandler
    import threading
    # a stuck collective must leave evidence: dump every thread's stack (and what the engine on this rank has done so
    # far) and exit instead of waiting for the caller
    limit = int(os.environ.get("GLLM_TP_CHECK_TIMEOUT", "420"))
    faulthandler.dump_traceback_later(limit, exit=True)

    def _where():
        llm = globals().get("_LIVE_LLM")
        if llm is not None and llm.worker is not None and llm.worker.runner is not None:
            w = llm.worker
            print(f"[stall rank {os.environ.get('RANK')}] runner steps {w.runner.stats['steps']} graph_steps "
                  f"{w.runner.stats['graph_steps']} queued peer batches {len(w.peer_batches)} pending {len(w.pending)} "
                  f"batch_counter {w.batch_counter}", flush=True)
    t = threading.Timer(max(limit - 5, 1), _where)
    t.daemon = True
    t.start()
    rank, local, world = int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(local)
    from gllm_b200.parallel import state as ps
    ps.init_dist(1, world, rank, local, os.environ.get("MASTER_ADDR", "127.0.0.1"),
                 int(os.environ.get("MASTER_PORT", "29500")) + 1)
    from gllm_b200.ops import ref, sm100
    from gllm_b200.parallel.fused import FusedTPComm
    from gllm_b200.parallel.tp import TPComm
    dev = torch.device("cuda", local)
    H, K, N2 = 1024, 512, 768
    def log(*a):
        if rank == 0:
            print("[tp_check]", *a, flush=True)
    log("dist ready")
    fused = FusedTPComm(max_tokens=1024, hidden_size=H, device=dev)
    base = TPComm(sm100)
    log("symmetric buffers ready")
    ok = True
    def op_level(T, tag=""):
        nonlocal ok
        torch.manual_seed(100 + T)  # same on every rank
        x_full = (torch.randn(T, H, device=dev) * 0.5).bfloat16()         # replicated "embedding" output
        nw0 = (1 + 0.1 * torch.randn(H, device=dev)).bfloat16()
        nw1 = (1 + 0.1 * torch.randn(H, device=dev)).bfloat16()
        w_col = (torch.randn(world, N2, H, device=dev) * 0.05).bfloat16()[rank]     # column-parallel shard
        w_row = (torch.randn(world, H, N2, device=dev) * 0.05).bfloat16()[rank]     # row-parallel shard
        w_col2 = (torch.randn(world, N2, H, device=dev) * 0.05).bfloat16()[rank]
        # ---- baseline (NCCL) ----
        h, res = base.first_norm(x_full.clone(), nw0, 1e-6)
        res = res.clone()
        a = base.col_linear(h, w_col)
        h2, res = base.row_linear_add_norm(a, w_row, res, nw1, 1e-6)
        y_ref = base.col_linear(h2, w_col2)
        torch.cuda.synchronize()
        log(f"T={T}: baseline done")
        # ---- fused ----
        for rep in range(3):  # repeated: exercises parity / epoch bookkeeping
            fused.begin_forward(T)
            hf, resf = fused.first_norm(x_full.clone(), nw0, 1e-6)
            torch.cuda.synchronize(); log(f"T={T} rep={rep}: first_norm ok")
            af = fused.col_linear(hf, w_col)
            torch.cuda.synchronize(); log("  ag-gemm ok")
            hf2, resf = fused.row_linear_add_norm(af, w_row, resf, nw1, 1e-6)
            torch.cuda.synchronize(); log("  gemm-rs + reduce_norm ok")
            y = fused.col_linear(hf2, w_col2)
            hf2m = fused.materialize(hf2).clone()
            torch.cuda.synchronize(); log("  second ag-gemm ok")
            e1 = ((af.float() - a.float()).norm() / a.float().norm()).item()
            e2 = ((hf2m.float() - h2.float()).norm() / h2.float().norm()).item()
            e3 = ((y.float() - y_ref.float()).norm() / y_ref.float().norm()).item()
            r0 = rank * fused.rpr
            rv = fused._rows_valid()
            if fused.small:  # tiny forwards run the replicated (NCCL) strategy
                r0, rv = 0, T
            e4 =((resf[:rv].float() - res[r0:r0 + rv].float()).norm() / (res[r0:r0 + rv].float().norm() + 1e-9)).item() if rv else 0.0
            if max(e1, e2, e3, e4) > 2e-2:
                ok = False
                print(f"[rank {rank}] {tag}T={T} rep={rep} MISMATCH {e1:.4f} {e2:.4f} {e3:.4f} {e4:.4f}", flush=True)
        dist.barrier()

    for T in (1000, 37, 256, 5):
        op_level(T)
    if fused.mc_base:
        # the same dataflow with the decode-sized all-reduce forced onto the NVLS (multimem, in-switch reduction)
        # kernel instead of the LL peer-store one
        keep_rows, fused.nvls_min_peer_rows = fused.nvls_min_peer_rows, 0
        calls0 = fused.nvls_calls
        for T in (37, 5, 64):
            op_level(T, "nvls ")
        if fused.nvls_calls == calls0:
            ok = False
            print(f"[rank {rank}] NVLS path did not run", flush=True)
        fused.nvls_min_peer_rows = keep_rows
        log(f"NVLS all-reduce: {fused.nvls_calls - calls0} calls checked")
    else:
        log("no multicast mapping on this box: NVLS all-reduce not exercised")
    # MoE-style partial push
    T = 200
    torch.manual_seed(7)
    part = (torch.randn(world, T, H, device=dev) * 0.3).bfloat16()
    nw = (1 + 0.1 * torch.randn(H, device=dev)).bfloat16()
    x0 = (torch.randn(T, H, device=dev) * 0.5).bfloat16()
    hb, rb = base.first_norm(x0.clone(), nw, 1e-6)
    rb = rb.clone()
    hb2, rb = base.reduce_add_norm(part[rank].clone(), rb, nw, 1e-6)
    fused.begin_forward(T)
    hf, rf = fused.first_norm(x0.clone(), nw, 1e-6)
    hf2, rf = fused.reduce_add_norm(part[rank].clone(), rf, nw, 1e-6)
    hf2 = fused.materialize(hf2).clone()
    torch.cuda.synchronize()
    e = ((hf2.float() - hb2.float()).norm() / hb2.float().norm()).item()
    if e > 2e-2:
        ok = False
        print(f"[rank {rank}] partial push mismatch {e}", flush=True)
    dist.barrier()

    # ---- expert-parallel all-to-all (dispatch -> grouped GEMMs with return-push epilogue -> combine) ----
    from gllm_b200.layers.moe import FusedMoE

    class _Blk(torch.nn.Module):
        shared = None

        def __init__(self, ex):
            super().__init__()
            self.experts = ex

        def forward(self, h, tpc):
            return self.experts(h, tpc)

    E, topk, inter = 8 if world <= 8 else world, 2, 256
    ex = FusedMoE(E, topk, H, inter, torch.bfloat16, dev)
    torch.manual_seed(99)
    ex.router_w.data.copy_((torch.randn(E, H, device=dev) * 0.2).bfloat16())
    for e in range(E):
        g = (torch.randn(inter, H, device=dev) * 0.05).bfloat16()
        u = (torch.randn(inter, H, device=dev) * 0.05).bfloat16()
        d = (torch.randn(H, inter, device=dev) * 0.05).bfloat16()
        ex.load_expert(e, g, u, d)
    blk = _Blk(ex)
    for T in (300, 129, 1000):
        torch.manual_seed(500 + T)
        x0 = (torch.randn(T, H, device=dev) * 0.5).bfloat16()
        hb, rb = base.first_norm(x0.clone(), nw, 1e-6)
        hb2, rb2 = base.moe_add_norm(blk, hb, rb.clone(), nw, 1e-6)
        for rep in range(3):
            fused.begin_forward(T)
            hf, rf = fused.first_norm(x0.clone(), nw, 1e-6)
            assert fused.can_a2a(blk)
            hf2, rf = fused.moe_add_norm(blk, hf, rf, nw, 1e-6)
            hf2, rf = fused.moe_add_norm(blk, hf2, rf, nw, 1e-6)   # two layers: both pool parities
            hf2 = fused.materialize(hf2).clone()
            torch.cuda.synchronize()
            if rep == 0:
                hb3, _ = base.moe_add_norm(blk, hb2, rb2.clone(), nw, 1e-6)
            e = ((hf2.float() - hb3.float()).norm() / hb3.float().norm()).item()
            log(f"ep a2a T={T} rep={rep}: rel err {e:.4f}")
            if not e < 3e-2:
                ok = False
                print(f"[rank {rank}] ep a2a mismatch T={T} rep={rep}: {e}", flush=True)
        dist.barrier()

    # ---- engine level ----
    from gllm_b200 import LLM
    from gllm_b200.models.presets import tiny
    cfgs = {
        "qwen3": tiny("Qwen3ForCausalLM", hidden_size=512, num_hidden_layers=3, num_attention_heads=8,
                      num_key_value_heads=2, head_dim=64, intermediate_size=1024, vocab_size=2048,
                      torch_dtype="bfloat16"),
        "mixtral-ep": tiny("MixtralForCausalLM", hidden_size=512, num_hidden_layers=3, num_attention_heads=8,
                           num_key_value_heads=2, head_dim=64, intermediate_size=256, vocab_size=2048,
                           num_local_experts=8, num_experts_per_tok=2, torch_dtype="bfloat16"),
    }
    prompts = [[5, 9, 100, 7], list(range(20, 190)), [77] * 33, [3, 1, 4, 1, 5, 9, 2, 6]]
    # the runner keeps every step's last-token logits (all ranks: collective)
    os.environ["GLLM_KEEP_LOGITS"] = os.environ.get("GLLM_TP_CHECK_LOGITS", "1")
    keep = os.environ["GLLM_KEEP_LOGITS"] == "1"
    n_out = 8
    for name, cfg in cfgs.items():
        toks, logs = {}, {}
        for mode in ("nccl", "fused"):
            torch.manual_seed(4321 + rank)
            llm = LLM(cfg, load_format="dummy", tp_size=world, maxp=128, maxd=64, max_cuda_graph_bs=8,
                      num_gpu_pages=256, model_max_length=512, log_stats=False, tp_mode=mode, launch_mode="inproc",
                      async_schedule=os.environ.get("GLLM_TP_CHECK_ASYNC", "1") == "1")
            globals()["_LIVE_LLM"] = llm
            outs = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True)
            if rank == 0:
                toks[mode] = [s.token_ids[len(p):] for s, p in zip(outs, prompts)]
                assert llm.worker.runner.stats["graph_steps"] > 0
                # per sequence: the logits rows in emission order
                per_seq = {s.seq_id: [] for s in outs}
                for ids, lg in llm.worker.runner.logit_log:
                    for row, sid in enumerate(ids):
                        per_seq[sid].append(lg[row])
                logs[mode] = [per_seq[s.seq_id] for s in outs]
            if mode == "fused" and name == "mixtral-ep":
                assert llm.worker.runner.tpc.ep is not None, "EP all-to-all path did not run"
            llm.close()
        if rank == 0 and not keep:
            agree = sum(a == b for x, y in zip(toks["nccl"], toks["fused"]) for a, b in zip(x, y))
            print(name, f"token agreement {agree}/{n_out * len(prompts)} (logits check disabled)", flush=True)
        if rank == 0 and keep:
            # Logits-based criterion: as long as a sequence's tokens agree between the two modes its inputs are
            # identical, so the last-token logits of that step must agree to bf16 accumulation-order noise; and
            # where the greedy tokens first differ, it has to be a genuine near-tie in BOTH modes' logits.
            worst, checked, flips = 0.0, 0, 0
            for si, (tn, tf) in enumerate(zip(toks["nccl"], toks["fused"])):
                for j in range(n_out):
                    ln, lf = logs["nccl"][si][j], logs["fused"][si][j]
                    scale = float(ln.abs().max()) + 1e-6
                    err = float((ln - lf).abs().max()) / scale
                    worst = max(worst, err)
                    checked += 1
                    if err > 4e-2:
                        ok = False
                        print(f"{name}: seq {si} step {j}: logits differ, max-abs err {err:.4f} of the row scale",
                              flush=True)
                    if tn[j] != tf[j]:
                        flips += 1
                        gap = float(ln[tn[j]] - ln[tf[j]]) / scale      # >= 0: tn[j] is nccl's argmax
                        if gap > 4e-2:
                            ok = False
                            print(f"{name}: seq {si} step {j}: tokens {tn[j]} vs {tf[j]} differ without a near-tie "
                                  f"(gap {gap:.4f} of the row scale)", flush=True)
                        break       # later steps run on different inputs
            print(f"{name}: {checked} logits rows compared on identical inputs, worst max-abs err {worst:.4f} of the "
                  f"row scale, {flips} greedy near-tie flips", flush=True)
            if [x[0] for x in toks["nccl"]] != [y[0] for y in toks["fused"]] and name == "qwen3" and world <= 4:
                print(name, "first tokens differ:", toks["nccl"], toks["fused"], flush=True)

    # ---- vocab-parallel sampling at engine level: sampled requests never gather the [E, V] logits ----
    os.environ["GLLM_KEEP_LOGITS"] = "0"
    llm = LLM(cfgs["qwen3"], load_format="dummy", tp_size=world, maxp=128, maxd=64, max_cuda_graph_bs=8,
              num_gpu_pages=256, model_max_length=512, log_stats=False, tp_mode="fused", launch_mode="inproc")
    outs = llm.generate(tokens=prompts, output_lens=[n_out] * len(prompts), ignore_eos=True,
                        temperature=[0.0, 0.8, 1.0, 0.7], top_p=[1.0, 0.9, 1.0, 0.5], top_k=[1, 8, 0, 0],
                        repetition_penalty=[1.0, 1.2, 1.0, 1.0])
    if rank == 0:
        st = llm.worker.runner.stats
        if st.get("vp_sample_steps", 0) == 0 or any(len(s.token_ids) != len(p) + n_out for s, p in zip(outs, prompts)) \
                or max(max(s.token_ids) for s in outs) >= 2048:
            ok = False
            print("vocab-parallel sampling at engine level failed", st, flush=True)
    llm.close()
    t = torch.tensor([1 if ok else 0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    if rank == 0:
        print("TP_CHECK_OK" if t.item() == 1 else "TP_CHECK_FAILED", flush=True)
    dist.barrier()
    sys.stdout.flush()
    fused.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
