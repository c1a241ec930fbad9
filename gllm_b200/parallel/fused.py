"""Fused tensor-parallel strategy (the product path for tp > 1, pp == 1): token-sharded activations,
row-parallel GEMM ⊕ reduce-scatter and all-gather ⊕ column-parallel GEMM over NVLink peer memory.

Per block (kernels: csrc/gemm/gemm_bf16.cu hooks + csrc/comm/tp_fused.cu):

    attn out ──► O-proj GEMM, epilogue stores partial tiles into the OWNER rank's staging slot (P2P st)
             ──► rs_reduce_norm on the owner: wait tile counters, sum tp partials (fixed order), + residual
                 shard, RMSNorm, push normed rows into EVERY rank's gather buffer, raise epoch flags
             ──► gate/up GEMM whose TMA producer warp waits (ld.acquire.sys) for the row shards covering
                 its M tile ... (same again for down-proj / next layer's QKV)

Symmetric buffers come from `torch.distributed._symmetric_memory` (CUDA VMM + handle exchange); all
synchronisation state (expected counters, epochs) lives in device memory so CUDA graphs can replay it.
Reference behaviour replaced: GEMM -> NCCL all_reduce -> fused_add_rms_norm on replicated activations
(gllm/layers/linear.py:247-250, gllm/dist_utils.py:253-256).
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist

from gllm_b200.ops import lib as _lib
from gllm_b200.ops.lib import EpArgs, GemmComm, LLArgs, NvlsArgs, ReduceNormArgs, launch
from gllm_b200.parallel import state as ps
from gllm_b200.parallel.tp import TPComm
from gllm_b200.utils.logging import logger


_ONESHOT = os.environ.get("GLLM_TP_ONESHOT", "1") != "0"
MAX_BLOCKS = 256   # kMaxBlocks in csrc/comm/tp_fused.cu (128-row blocks per gather buffer)
# SMALL_T: row capacity of the decode-sized all-reduce buffers; forwards with <= small_threshold(tp) tokens run on
# replicated rows + the one-kernel all-reduce⊕add⊕norm instead of the token-sharded GEMM⊕RS / AG⊕GEMM dataflow (see
# begin_forward; sweep with benchmarks/tp_small_t_sweep.py). GLLM_TP_SMALL_T=<n> sets both; GLLM_TP_SMALL_T=auto
# keeps the 64-row buffers and scales the threshold with the LL variant's incoming traffic, (tp-1)*T rows.
_SMALL_T_ENV = os.environ.get("GLLM_TP_SMALL_T", "64")
SMALL_T = 64 if _SMALL_T_ENV == "auto" else int(_SMALL_T_ENV)


def small_threshold(tp: int) -> int:
    if _SMALL_T_ENV != "auto":
        return SMALL_T
    return max(8, min(SMALL_T, 112 // max(tp - 1, 1)))


class FusedTPComm(TPComm):
    fused = True

    def __init__(self, max_tokens: int, hidden_size: int, dtype=torch.bfloat16, device=None, **_):
        from gllm_b200.ops import sm100
        super().__init__(sm100)
        assert dtype == torch.bfloat16, "fused TP path is bf16"
        import torch.distributed._symmetric_memory as symm
        st = ps.get_state()
        self.group = st.tp_group
        self.device = torch.device(device)
        tp = self.tp_size
        self.H = hidden_size
        self.max_tokens = max_tokens
        self.rpr_max = (max_tokens + tp - 1) // tp
        t_pad = self.rpr_max * tp
        L = _lib.load()
        self.L = L
        # ---- one symmetric blob: [stage x2][ag x3][cnt x2][flags x3] ----
        stage_bytes = tp * self.rpr_max * hidden_size * 2
        ag_bytes = t_pad * hidden_size * 2
        self.off_stage = [0, stage_bytes]
        self.off_ag = [2 * stage_bytes + i * ag_bytes for i in range(3)]
        base_sync = 2 * stage_bytes + 3 * ag_bytes
        self.off_cnt = [base_sync, base_sync + 64]
        self.off_flag = [base_sync + 128 + 4 * MAX_BLOCKS * i for i in range(3)]
        total = base_sync + 128 + 4 * MAX_BLOCKS * 3
        assert t_pad <= 128 * MAX_BLOCKS
        total = (total + 255) // 256 * 256
        # LL slots of the one-shot all-reduce: [parity][src][SMALL_T rows][H/2] x 8 bytes
        ll_bytes = tp * SMALL_T * hidden_size * 4
        self.off_ll = [total, total + ll_bytes]
        total += 2 * ll_bytes
        # NVLS (multimem) all-reduce: [parity][SMALL_T rows][H] bf16 partial rows + [tp][SMALL_T] epoch flags
        nv_bytes = SMALL_T * hidden_size * 2
        self.off_nv = [total, total + nv_bytes]
        self.off_nv_flags = total + 2 * nv_bytes
        total += 2 * nv_bytes + (tp * SMALL_T * 4 + 255) // 256 * 256
        self.blob = symm.empty(total, dtype=torch.uint8, device=self.device)
        self.blob.zero_()
        self.hdl = symm.rendezvous(self.blob, self.group.group_name)
        self.peer_base = [int(p) for p in self.hdl.buffer_ptrs]
        # multicast mapping of the same allocation (NVSwitch + driver support): in-switch reduction for the
        # decode-sized all-reduce. GLLM_TP_NVLS=0 keeps the LL (peer-store) variant everywhere;
        # GLLM_TP_NVLS_MIN_PEER_ROWS: NVLS from (tp-1)*T >= this many incoming rows (below, LL's single hop wins)
        self.mc_base = 0
        try:
            # opt-in (GLLM_TP_NVLS=1): numerically validated against NCCL (tests/mp_tp_check.py), not yet tuned
            # against the LL variant at every (tp, T)
            if os.environ.get("GLLM_TP_NVLS", "0") == "1" and getattr(self.hdl, "has_multicast_support", True):
                self.mc_base = int(self.hdl.multicast_ptr or 0)
        except Exception:  # noqa: BLE001
            self.mc_base = 0
        self.nvls_min_peer_rows = int(os.environ.get("GLLM_TP_NVLS_MIN_PEER_ROWS", "96"))
        self.nvls_calls = 0
        assert len(self.peer_base) == tp
        self.local_base = self.peer_base[self.tp_rank]
        assert self.local_base == self.blob.data_ptr()
        n_state = L.gllm_tp_state_bytes()
        self.state = torch.zeros(n_state, dtype=torch.uint8, device=self.device)
        # TpState layout: rs_expected[2][8] | ag_epoch[3] | ticket[4] | pad[9] | ag_expected[3][MAX_BLOCKS] (u32)
        assert n_state == 128 + 3 * MAX_BLOCKS * 4, n_state
        self.ag_expected_ptr = [self.state.data_ptr() + 128 + 4 * MAX_BLOCKS * i for i in range(3)]
        # device tables of peer pointers for the row-push kernel
        self.stage_tbl = [torch.tensor([b + self.off_stage[p] for b in self.peer_base], dtype=torch.int64,
                                       device=self.device) for p in range(2)]
        self.cnt_tbl = [torch.tensor([b + self.off_cnt[p] for b in self.peer_base], dtype=torch.int64,
                                     device=self.device) for p in range(2)]
        self.residual_buf = torch.zeros(self.rpr_max, hidden_size, dtype=dtype, device=self.device)
        torch.cuda.synchronize()
        dist.barrier(group=self.group)
        self.T = 0
        self.rpr = 0
        self.rs_call = 0
        self.ag_call = 0
        self.small = False
        self.oneshot = False
        self.cur_ag = None  # (ag_idx, tensor view) produced by the last reduce_norm
        self.ep = None      # expert-parallel all-to-all buffers, created by the first MoE block
        self.ep_call = 0
        logger.info("fused TP: %d MB symmetric buffer per rank, peers mapped over NVLink%s", total >> 20,
                    ", NVLS multicast mapping available" if self.mc_base else ", no multicast mapping (LL all-reduce)")

    # -------------------------------------------------------------------------------------------
    def begin_forward(self, num_tokens: int):
        assert num_tokens <= self.max_tokens
        # Tiny decode batches are latency bound: the swap-AB weight-streaming GEMMs + one NCCL
        # all-reduce beat the sharded dataflow there, so such forwards run the baseline strategy; everything
        # else runs fused.
        tp = self.tp_size
        # (a forward in which some rank would own no rows of the token-sharded layout stays on the replicated form)
        self.small = num_tokens <= small_threshold(tp) or \
            (num_tokens <= SMALL_T and (tp - 1) * ((num_tokens + tp - 1) // tp) >= num_tokens)
        # decode-sized forwards: one-shot all-reduce fused into the GEMM epilogue + reduce/add/norm kernel
        # (every rank pushes its partial rows to every rank); needs T rows per source in the staging slots
        self.oneshot = self.small and _ONESHOT and num_tokens <= self.rpr_max
        self.T = num_tokens
        self.rpr = (num_tokens + self.tp_size - 1) // self.tp_size
        self.rs_call = 0
        self.ag_call = 0
        self.cur_ag = None

    def _rows_valid(self) -> int:
        return max(0, min(self.rpr, self.T - self.tp_rank * self.rpr))

    def _next_ag_idx(self) -> int:
        i = 2 if self.ag_call == 0 else (self.ag_call - 1) % 2
        self.ag_call += 1
        return i

    def _ag_view(self, idx: int) -> torch.Tensor:
        off = self.off_ag[idx]
        return self.blob[off: off + self.T * self.H * 2].view(torch.bfloat16).view(self.T, self.H)

    def _reduce_norm(self, parity: int, n_tiles, local_x, residual_in: bool, norm_w, eps: float,
                     bcast: bool = False, push_x=None):
        """bcast=True: one-shot all-reduce form — every rank received every rank's partial for ALL T rows and
        reduces them itself; the normed rows stay local (no gather push) and the residual is replicated."""
        ag_idx = self._next_ag_idx()
        a = ReduceNormArgs()
        a.stage = self.local_base + self.off_stage[parity]
        a.cnt = self.local_base + self.off_cnt[parity]
        for s in range(self.tp_size):
            a.n_tiles[s] = n_tiles
        a.local_x = local_x.data_ptr() if local_x is not None else None
        a.local_ld = local_x.stride(0) if local_x is not None else 0
        a.residual = self.residual_buf.data_ptr()
        a.residual_in = 1 if residual_in else 0
        a.norm_w = norm_w.data_ptr()
        for p in range(self.tp_size):
            a.ag_peers[p] = self.peer_base[p] + self.off_ag[ag_idx]
            a.flag_peers[p] = self.peer_base[p] + self.off_flag[ag_idx]
        a.unnormed_out = None
        a.st = self.state.data_ptr()
        a.parity, a.ag_idx, a.tp, a.rank = parity, ag_idx, self.tp_size, self.tp_rank
        a.rows_per_rank, a.rows_valid, a.H, a.eps = self.rpr, self._rows_valid(), self.H, float(eps)
        a.T = self.T
        a.bcast = 1 if bcast else 0
        if bcast:
            a.rows_per_rank = a.rows_valid = self.T
        if push_x is not None:
            assert bcast and push_x.stride(1) == 1
            a.push_x, a.push_ld = push_x.data_ptr(), push_x.stride(0)
            for p in range(self.tp_size):
                a.stage_peers[p] = self.peer_base[p] + self.off_stage[parity]
                a.cnt_peers[p] = self.peer_base[p] + self.off_cnt[parity]
        launch("gllm_rs_reduce_norm", a)
        h = self._ag_view(ag_idx)
        if bcast:
            self.cur_ag = None  # all rows were written by this rank's own kernel: nothing to gate on
            return h, self.residual_buf[: self.T]
        self.cur_ag = (ag_idx, h)
        return h, self.residual_buf[: self.rpr]

    def _ag_comm(self, x: torch.Tensor) -> Optional[GemmComm]:
        """GemmComm that gates the A operand on the gather flags, if x is the live gather buffer."""
        if self.cur_ag is None or x.data_ptr() != self.cur_ag[1].data_ptr():
            return None
        idx = self.cur_ag[0]
        c = GemmComm()
        c.a_ready = self.local_base + self.off_flag[idx]
        c.a_expected = self.ag_expected_ptr[idx]
        num_m = (self.T + 127) // 128
        c.m_rot = ((self.tp_rank * self.rpr) // 128) % max(num_m, 1)  # start with this rank's own rows
        c.rs_world = 0
        return c

    # -------------------------------------------------------------------------------------------
    def first_norm(self, x: torch.Tensor, norm_w: torch.Tensor, eps: float):
        """Embedding output (replicated) -> (normed gather buffer, residual shard)."""
        if self.small:
            if self.oneshot:
                return self._reduce_norm(0, 0, x, False, norm_w, eps, bcast=True)
            return super().first_norm(x, norm_w, eps)
        return self._reduce_norm(0, 0, x, False, norm_w, eps)

    def stage_exit(self, residual):
        """Pipeline stage boundary: inside a stage the residual stream is token-sharded (each rank owns `rpr` rows);
        the next stage receives it replicated, so gather the shards (once per stage and step, on NCCL)."""
        if residual is None or self.small:
            return residual
        full = ps.tp_all_gather_first_dim(residual[: self.rpr].contiguous())
        return full[: self.T]

    def materialize(self, h: torch.Tensor) -> torch.Tensor:
        """Make the gather buffer safe to read by a kernel that does not understand the flags."""
        if not self.small and self.cur_ag is not None and h.data_ptr() == self.cur_ag[1].data_ptr():
            idx = self.cur_ag[0]
            launch("gllm_wait_ag_flags", self.local_base + self.off_flag[idx], self.state.data_ptr(), idx, self.T)
        return h

    def col_linear(self, x, w, bias=None):
        from gllm_b200.ops import sm100
        comm = None if self.small else self._ag_comm(x)
        if comm is None:
            return sm100.linear(x, w, bias)
        return sm100.linear(x, w, bias, comm=comm)

    def col_linear_silu_mul(self, x, w_interleaved):
        from gllm_b200.ops import sm100
        comm = None if self.small else self._ag_comm(x)
        if comm is None:
            return sm100.linear_silu_mul(x, w_interleaved)
        return sm100.linear_silu_mul(x, w_interleaved, comm=comm)

    def row_linear_add_norm(self, x, w, residual, norm_w, eps, bias=None, delta=None):
        assert delta is None, "LoRA deltas run on the NCCL strategy (the partial output is never materialised here)"
        from gllm_b200.ops import sm100
        if self.small:
            # decode-sized T: best local GEMM for the shape (swap-AB / split-K), then the one-kernel
            # all-reduce ⊕ add ⊕ norm (reduce_add_norm below); TPComm.row_linear_add_norm does exactly that
            return super().row_linear_add_norm(x, w, residual, norm_w, eps, bias)
        parity = self.rs_call % 2
        self.rs_call += 1
        t, n = x.shape[0], w.shape[0]
        assert t == self.T and n == self.H
        bcast = self.small
        c = GemmComm()
        c.a_ready = None
        c.rs_world, c.rs_rank, c.rows_per_rank, c.rs_inc = self.tp_size, self.tp_rank, (t if bcast else self.rpr), 1
        c.rs_bcast = 1 if bcast else 0
        for p in range(self.tp_size):
            c.peer_out[p] = self.peer_base[p] + self.off_stage[parity]
            c.peer_cnt[p] = self.peer_base[p] + self.off_cnt[parity]
        # the epilogue writes into the peers' staging slots; `out` is only a shape carrier
        dummy = self.blob[self.off_stage[parity]: self.off_stage[parity] + 16].view(torch.bfloat16)
        sm100.linear(x, w, bias if self.tp_rank == 0 else None, out=_FakeOut(t, n, dummy), comm=c)
        r0 = 0 if bcast else self.tp_rank * self.rpr
        ws = sm100._smallm_workspace(x.device)[0]
        n_tiles = self.L.gllm_gemm_bf16_tiles_covering(t, n, x.shape[1], 0, sm100._FORCE_BN, r0,
                                                       t if bcast else min(r0 + self.rpr, t), ws.numel() * 4,
                                                       sm100._SPLITK_MAX_TILES)
        return self._reduce_norm(parity, n_tiles, None, residual is not None, norm_w, eps, bcast=bcast)

    def reduce_add_norm(self, partial, residual, norm_w, eps):
        if self.small:
            if not self.oneshot or partial.dtype != torch.bfloat16:
                return super().reduce_add_norm(partial, residual, norm_w, eps)
            # one-shot all-reduce: push the partial rows to every rank, sum all tp partials locally, + residual,
            # RMSNorm — one kernel instead of NCCL all-reduce + add/norm
            parity = self.rs_call % 2
            self.rs_call += 1
            assert partial.shape[0] == self.T and partial.shape[1] == self.H and partial.stride(1) == 1
            if self.H // 8 > 1024:   # rows wider than one CTA: counter-based one-shot form
                return self._reduce_norm(parity, self.T, None, residual is not None, norm_w, eps, bcast=True,
                                         push_x=partial)
            h = self._ag_view(self._next_ag_idx())
            if self.mc_base and (self.tp_size - 1) * self.T >= self.nvls_min_peer_rows:
                # in-switch reduction: H*2 bytes per row each way instead of (tp-1)*H*4 bytes of LL slots
                n = NvlsArgs()
                n.x, n.ldx = partial.data_ptr(), partial.stride(0)
                n.residual, n.residual_in = self.residual_buf.data_ptr(), 1 if residual is not None else 0
                n.norm_w, n.out = norm_w.data_ptr(), h.data_ptr()
                n.buf_local = self.local_base + self.off_nv[parity]
                n.buf_mc = self.mc_base + self.off_nv[parity]
                n.flags_mc = self.mc_base + self.off_nv_flags
                n.flags_local = self.local_base + self.off_nv_flags
                n.st = self.state.data_ptr()
                n.tp, n.rank, n.T, n.H, n.row_cap, n.eps = (self.tp_size, self.tp_rank, self.T, self.H, SMALL_T,
                                                            float(eps))
                launch("gllm_nvls_allreduce_norm", n)
                self.nvls_calls += 1
                self.cur_ag = None
                return h, self.residual_buf[: self.T]
            a = LLArgs()
            a.x, a.ldx = partial.data_ptr(), partial.stride(0)
            a.residual, a.residual_in = self.residual_buf.data_ptr(), 1 if residual is not None else 0
            a.norm_w, a.out = norm_w.data_ptr(), h.data_ptr()
            for p in range(self.tp_size):
                a.ll_peers[p] = self.peer_base[p] + self.off_ll[parity]
            a.st = self.state.data_ptr()
            a.tp, a.rank, a.T, a.H, a.row_cap, a.eps = self.tp_size, self.tp_rank, self.T, self.H, SMALL_T, float(eps)
            launch("gllm_ll_allreduce_norm", a)
            self.cur_ag = None
            return h, self.residual_buf[: self.T]
        parity = self.rs_call % 2
        self.rs_call += 1
        assert partial.shape[0] == self.T and partial.shape[1] == self.H and partial.stride(1) == 1
        launch("gllm_push_partial_rows", partial.data_ptr(), partial.stride(0), self.T, self.H, self.tp_rank, self.rpr,
               self.stage_tbl[parity].data_ptr(), self.cnt_tbl[parity].data_ptr())
        return self._reduce_norm(parity, self._rows_valid(), None, residual is not None, norm_w, eps)

    def close(self):
        """Drop the symmetric-memory mappings (collective: every rank of the group, peers alive)."""
        torch.cuda.synchronize()
        dist.barrier(group=self.group)
        self.ep = None
        self.cur_ag = None
        self.hdl = None
        self.blob = None

    # -------------------------------------------------------------------------------------------
    # expert-parallel all-to-all (csrc/comm/ep_a2a.cu)
    # -------------------------------------------------------------------------------------------
    def _ep_setup(self, experts):
        """Collective (every rank reaches its first MoE block together, in the eager profile run)."""
        import torch.distributed._symmetric_memory as symm
        tp, H, k = self.tp_size, self.H, experts.top_k
        per = experts.num_experts // tp
        e_local_max = experts.num_experts - (tp - 1) * per
        r_max = self.max_tokens * min(k, e_local_max)
        r_max = (r_max + 127) // 128 * 128
        comb_rows = self.rpr_max * k
        sz = {"recv_x": r_max * H * 2, "recv_e": r_max * 4, "recv_src": r_max * 4, "comb": comb_rows * H * 2,
              "ctrl": 256}
        off, cur = [], 0
        for _ in range(2):
            o = {}
            for name, n in sz.items():
                o[name] = cur
                cur += (n + 255) // 256 * 256
            off.append(o)
        blob = symm.empty(cur, dtype=torch.uint8, device=self.device)
        blob.zero_()
        hdl = symm.rendezvous(blob, self.group.group_name)
        bases = [int(p) for p in hdl.buffer_ptrs]
        state = torch.zeros(self.L.gllm_ep_state_bytes(), dtype=torch.uint8, device=self.device)
        args = []
        for par in range(2):
            a = EpArgs()
            for p in range(tp):
                a.recv_x[p] = bases[p] + off[par]["recv_x"]
                a.recv_e[p] = bases[p] + off[par]["recv_e"]
                a.recv_src[p] = bases[p] + off[par]["recv_src"]
                a.ctrl[p] = bases[p] + off[par]["ctrl"]
                a.comb[p] = bases[p] + off[par]["comb"]
            a.state = state.data_ptr()
            a.ep, a.rank, a.experts_per_rank, a.top_k, a.H, a.r_max = tp, self.tp_rank, per, k, H, r_max
            args.append(a)

        def view(par, name, dtype, shape):
            o = off[par][name]
            n = 1
            for d in shape:
                n *= d
            return blob[o: o + n * torch.empty((), dtype=dtype).element_size()].view(dtype).view(*shape)

        self.ep = dict(
            blob=blob, hdl=hdl, state=state, args=args, r_max=r_max, k=k,
            recv_x=[view(p, "recv_x", torch.bfloat16, (r_max, H)) for p in range(2)],
            recv_e=[view(p, "recv_e", torch.int32, (r_max, 1)) for p in range(2)],
            n_valid=[view(p, "ctrl", torch.int32, (1,)) for p in range(2)],
            out=torch.zeros(self.rpr_max, H, dtype=torch.bfloat16, device=self.device),
            row_dest=torch.zeros(r_max + 128 * (e_local_max + 1), dtype=torch.int64, device=self.device))
        torch.cuda.synchronize()
        dist.barrier(group=self.group)
        logger.info("EP all-to-all: %d MB symmetric pool per rank (%d rows x2)", cur >> 20, r_max)

    def can_a2a(self, block) -> bool:
        ex = getattr(block, "experts", None)
        return (not self.small and ex is not None and ex.use_ep and getattr(block, "shared", None) is None
                and ex.w13.is_cuda and ex.w13.dtype == torch.bfloat16 and ex.top_k <= 63)

    def moe_add_norm(self, block, h, residual, norm_w, eps):
        """MoE block + residual add + next RMSNorm. Routed experts only (no shared expert) and EP:
        dispatch -> grouped GEMMs whose epilogue returns the rows -> combine, all over peer memory."""
        if not self.can_a2a(block):
            return super().moe_add_norm(block, h, residual, norm_w, eps)
        from gllm_b200.ops import sm100_moe
        ex = block.experts
        if self.ep is None:
            self._ep_setup(ex)
        ep = self.ep
        assert ep["k"] == ex.top_k
        par = self.ep_call % 2
        self.ep_call += 1
        a = ep["args"][par]
        rv, r0 = self._rows_valid(), self.tp_rank * self.rpr
        if rv > 0:
            w, ids = ex.route(h[r0:r0 + rv])   # own rows of the gather buffer are local writes: no flag wait
            xs = h[r0:r0 + rv]
            launch("gllm_ep_dispatch", a, xs.data_ptr(), xs.stride(0), ids.data_ptr(), rv, n=0)
        else:
            w = None
            launch("gllm_ep_dispatch", a, None, 0, None, 0, n=0)

        def row_dest_fn(slot_pos, rows):
            rd = ep["row_dest"]
            assert rows <= rd.numel()
            launch("gllm_ep_row_dest", a, slot_pos.data_ptr(), rd.data_ptr(), rows, n=0)
            return rd

        sm100_moe.fused_experts(ep["recv_x"][par], ex.w13, ex.w2, None, ep["recv_e"][par], None,
                                n_valid=ep["n_valid"][par], row_dest_fn=row_dest_fn)
        out = ep["out"]
        launch("gllm_ep_combine", a, w.data_ptr() if w is not None else None, out.data_ptr(), rv, n=6)
        # `out` holds this rank's rows only; rs_reduce_norm indexes a full [T, H] tensor by global row
        shifted = _ShiftedRows(out, r0)
        return self._reduce_norm(0, 0, shifted, residual is not None, norm_w, eps)

    def row_linear(self, x, w, bias=None, delta=None):
        assert delta is None, "LoRA deltas run on the NCCL strategy"
        if self.small:
            return super().row_linear(x, w, bias)
        raise NotImplementedError("fused TP is used with pp_size == 1 (no un-normalised stage boundary)")


class _ShiftedRows:
    """Presents a rank-local [rows, H] tensor as if it were rows [r0, r0+rows) of a full tensor."""

    def __init__(self, t, r0):
        self._t, self._r0 = t, r0

    def stride(self, i):
        return self._t.stride(i)

    def data_ptr(self):
        return self._t.data_ptr() - self._r0 * self._t.stride(0) * self._t.element_size()


class _FakeOut:
    """Duck-typed `out=` for sm100.linear when the epilogue writes to peer memory instead."""

    def __init__(self, m, n, t):
        self.shape = (m, n)
        self._t = t

    def stride(self, i):
        return self.shape[1] if i == 0 else 1

    def data_ptr(self):
        return self._t.data_ptr()
