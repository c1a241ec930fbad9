"""Commit-able SASS listings of the hot sm_90a kernels (runs without a GPU):

    python tools/sass_dump.py            # writes profiles/sass/<kernel>.sass

One file per kernel named in BASELINE.json's north star (GEMMs, attention, fused collectives, MoE, sampling, norm /
rope), cut out of `cuobjdump -sass` of the in-tree library: instruction text only (no encodings), so the files stay
small and diff-able. `tools/sass_summary.py` counts the mnemonics over ALL kernels."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gllm_b200", "_C", "libgllm_b200.so")
OUT = os.path.join(ROOT, "profiles", "sass")
WANT = ["gemm_bf16_kernel<128, 0>", "gemm_bf16_kernel<256, 1>", "gemm_smallm_kernel", "gemm_fp8_block_kernel",
        "attn_prefill_tc_kernel<128, 64>", "attn_prefill_kernel<128>", "attn_decode_kernel<128>", "attn_merge_kernel",
        "mla_attn_kernel", "rs_reduce_norm_kernel<1>", "ll_allreduce_norm_kernel", "push_partial_rows_kernel",
        "ep_dispatch_kernel", "ep_combine_kernel", "rope_kv_kernel<4>", "rmsnorm_kernel<1, 1>",
        "silu_and_mul_kernel", "sample_kernel<__nv_bfloat16>", "vp_candidates_kernel<__nv_bfloat16>",
        "vp_final_kernel", "topk_softmax_kernel<8>", "grouped_topk_kernel<8>", "nvls_allreduce_norm_kernel", "moe_combine_kernel"]


def main():
    os.makedirs(OUT, exist_ok=True)
    raw = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    names = subprocess.run(["cu++filt"], input="\n".join(re.findall(r"Function : (\S+)", raw)), capture_output=True,
                           text=True).stdout.splitlines()
    blocks = re.split(r"\n\s*Function : \S+\n", "\n" + raw)[1:]
    done = []
    for name, body in zip(names, blocks):
        short = re.sub(r"^(void )?b200::", "", name)
        short = short.replace("(int)", "").replace("(bool)", "").replace("(bool)", "")
        short = re.sub(r"\([^()]*\)$", "", short)
        hit = [w for w in WANT if short == w or short.startswith(w + "(")]
        if not hit:
            continue
        lines = []
        for ln in body.splitlines():
            m = re.match(r"\s*/\*([0-9a-f]{4})\*/\s+(.*?)\s*;?\s*/\*", ln)
            if m:
                lines.append(f"/*{m.group(1)}*/  {m.group(2).strip()}")
        fn = re.sub(r"[^A-Za-z0-9_]+", "_", hit[0]).strip("_") + ".sass"
        with open(os.path.join(OUT, fn), "w") as f:
            f.write(f"// {name}\n// {len(lines)} instructions; cuobjdump -sass gllm_b200/_C/libgllm_b200.so (sm_90a)\n")
            f.write("\n".join(lines) + "\n")
        done.append((hit[0], len(lines)))
    for k, n in done:
        print(f"{k}: {n} instructions")
    missing = [w for w in WANT if w not in [d[0] for d in done]]
    if missing:
        print("not found:", missing)


if __name__ == "__main__":
    main()
