"""Control-plane IPC over ZeroMQ (reference: gllm/comm.py:34-190).

Channels (all PUSH/PULL, HWM 0):
    front-end -> driver      requests / aborts / control commands          (pickled IPCPackage)
    driver    -> front-end   sampled tokens / freed ids                    (pickled IPCPackage)
    driver    -> every peer  one scheduled micro-batch per message         (header + raw arrays)
    output rank -> driver    sampled tokens (and log-probs) of a finished micro-batch

Differences from the reference: a micro-batch travels as flat numpy buffers (`BatchArrays`),
not as pickled `Sequence` objects that every rank re-expands in Python; sends are issued from the
calling thread (zmq queues them on its IO thread) instead of a new Python thread per message
(gllm/comm.py:166-167), which also keeps per-socket ordering.
"""
from __future__ import annotations

import os
import pickle
import struct
import time
import uuid
from dataclasses import dataclass, field
from typing import List, Optional

import zmq

from gllm_b200.input_data import BatchArrays


@dataclass
class IPCPackage:
    """Front-end <-> driver message (reference: gllm/comm.py:21-31)."""
    schedule_lists: list = field(default_factory=list)   # new Sequence objects (front-end -> driver)
    abort_ids: list = field(default_factory=list)
    act_schedule_ids: list = field(default_factory=list)  # driver -> front-end
    next_tokens: list = field(default_factory=list)
    next_logprobs: Optional[list] = None   # aligned with next_tokens when some request asked for log-probs
    prompt_logprobs: Optional[dict] = None  # seq id -> its next prompt log-prob entries, in prompt order
    free_ids: list = field(default_factory=list)
    control_cmd: Optional[tuple] = None
    stats: Optional[dict] = None


def make_socket(ctx: zmq.Context, kind: int, addr: str, bind: bool) -> zmq.Socket:
    s = ctx.socket(kind)
    s.setsockopt(zmq.LINGER, 0)
    if kind == zmq.PUSH:
        s.setsockopt(zmq.SNDHWM, 0)
        s.setsockopt(zmq.SNDBUF, 64 << 20)
    else:
        s.setsockopt(zmq.RCVHWM, 0)
        s.setsockopt(zmq.RCVBUF, 64 << 20)
    if bind:
        s.bind(addr)
    else:
        s.connect(addr)
    return s


def ipc_base(tag: Optional[str] = None) -> str:
    tag = tag or uuid.uuid4().hex[:12]
    return f"ipc:///tmp/gllm_b200_{tag}"


class Comm:
    """One instance per process. `role` in {"frontend", "driver", "peer"} (a process can be both
    front-end and driver when the engine runs in-process: then the front-end channel is bypassed)."""

    def __init__(self, base: str, rank: int, world_size: int, output_rank: int, frontend: bool = False,
                 tcp_host: Optional[str] = None, port_base: int = 8002, master_addr: str = "127.0.0.1"):
        self.base, self.rank, self.world_size, self.output_rank = base, rank, world_size, output_rank
        self.frontend = frontend
        self.tcp_host, self.port_base, self.master_addr = tcp_host, port_base, master_addr
        self.ctx = None  # created in init(): the object is pickled into spawned workers first
        self.sock_fe_in = self.sock_fe_out = None
        self.batch_out: List[zmq.Socket] = []
        self.batch_in = None
        self.tok_in = self.tok_out = None
        self.ring_w = self.ring_r = None       # shared-memory batch ring (driver writes, peers read)

    # addresses ---------------------------------------------------------------------------------
    def _addr(self, name: str, idx: int = 0, bind: bool = False) -> str:
        if self.tcp_host is not None:
            # multi-node: deterministic port per channel (reference: zmq_port_base + rank). Every TCP endpoint is
            # BOUND on the master node (front-end / driver) and connected to from wherever the other side runs,
            # so no node needs to know a slave's address.
            table = {"fe_req": 0, "fe_out": 1, "tok": 2}
            port = self.port_base + (table[name] if name in table else 3 + idx)
            if bind:
                # Bind on the master's own address, not on every interface: the frames on these sockets are pickled
                # Python objects (control messages, token lists), so whoever can connect can execute code in the
                # engine. The trust boundary is the cluster network the master address lives on (DESIGN.md, "Trust
                # boundary of the control plane"); `--host 0.0.0.0` restores the reference's bind-everywhere.
                wide = self.tcp_host in ("", "0.0.0.0", "*")
                return f"tcp://{'*' if wide else (self.tcp_host or self.master_addr)}:{port}"
            return f"tcp://{self.master_addr}:{port}"
        return f"{self.base}_{name}_{idx}"

    def init(self):
        P, L = zmq.PUSH, zmq.PULL
        self.ctx = zmq.Context.instance()
        if self.frontend:
            self.sock_fe_out = make_socket(self.ctx, P, self._addr("fe_req"), bind=False)
            self.sock_fe_in = make_socket(self.ctx, L, self._addr("fe_out", bind=True), bind=True)
            return self
        tcp = self.tcp_host is not None
        ring = self.use_shm_ring()
        if ring:
            self.init_ring()
        if self.rank == 0:
            self.sock_fe_in = make_socket(self.ctx, L, self._addr("fe_req", bind=True), bind=True)
            self.sock_fe_out = make_socket(self.ctx, P, self._addr("fe_out"), bind=False)
            for r in range(1, self.world_size if not ring else 1):
                # ipc: the peer binds its inbox and the driver connects; tcp: the driver binds, the peer connects
                self.batch_out.append(make_socket(self.ctx, P, self._addr("batch", r, bind=tcp), bind=tcp))
            if self.output_rank != 0:
                self.tok_in = make_socket(self.ctx, L, self._addr("tok", bind=True), bind=True)
        else:
            if not ring:
                self.batch_in = make_socket(self.ctx, L, self._addr("batch", self.rank, bind=not tcp), bind=not tcp)
            if self.rank == self.output_rank:
                self.tok_out = make_socket(self.ctx, P, self._addr("tok"), bind=False)
        return self

    # front-end <-> driver ----------------------------------------------------------------------
    def send_frontend(self, pkg: IPCPackage):
        self.sock_fe_out.send(pickle.dumps(pkg, protocol=pickle.HIGHEST_PROTOCOL))

    def recv_frontend(self) -> List[IPCPackage]:
        out = []
        while self.sock_fe_in is not None and self.sock_fe_in.poll(timeout=0):
            out.append(pickle.loads(self.sock_fe_in.recv()))
        return out

    # driver -> peers -----------------------------------------------------------------------------
    # batch channel: ZeroMQ PUSH/PULL per peer, or (GLLM_BATCH_TRANSPORT=shm, single node, x86-64) one
    # shared-memory broadcast ring written once by the driver — see engine/shm_ring.py for the why
    def use_shm_ring(self) -> bool:
        import platform
        return (self.tcp_host is None and self.world_size > 1 and self.base.startswith("ipc://")
                and os.environ.get("GLLM_BATCH_TRANSPORT", "zmq") == "shm"
                and platform.machine() in ("x86_64", "AMD64"))

    def _ring_name(self) -> str:
        return os.path.basename(self.base[len("ipc://"):]) + "_ring"

    def init_ring(self):
        from gllm_b200.engine import shm_ring
        if self.rank == 0:
            cap = int(os.environ.get("GLLM_SHM_RING_MB", "32")) << 20
            self.ring_w = shm_ring.RingWriter(self._ring_name(), self.world_size - 1, cap)
        else:
            self.ring_r = shm_ring.RingReader(self._ring_name(), self.rank - 1)

    @staticmethod
    def _encode_batch(batch: BatchArrays) -> bytes:
        """u32 header length | pickled header | pad to 16 | packed arrays — ONE buffer per batch. (Two-frame
        zero-copy multipart sends cost ~35 % more per peer for the ~10 KB decode batches that dominate.)"""
        hdr, bufs = batch.to_wire()
        h = pickle.dumps(hdr, protocol=pickle.HIGHEST_PROTOCOL)
        head = struct.pack("<I", len(h)) + h
        return b"".join((head, b"\0" * (-len(head) % 16), memoryview(bufs[0])))

    @staticmethod
    def _decode_batch(buf) -> BatchArrays:
        (n,) = struct.unpack_from("<I", buf, 0)
        hdr = pickle.loads(buf[4:4 + n])
        off = (4 + n + 15) // 16 * 16
        return BatchArrays.from_wire(hdr, [buf[off:]])

    def send_batch(self, batch: BatchArrays, ranks: Optional[List[int]] = None):
        if self.ring_w is not None:
            assert ranks is None
            self.ring_w.send(self._encode_batch(batch), 0)
            return
        if not self.batch_out:
            return
        msg = b"B" + self._encode_batch(batch)
        copy = len(msg) < (64 << 10)      # small: let zmq copy; large (prefill, pixel payloads): zero-copy
        for r, s in enumerate(self.batch_out, start=1):
            if ranks is None or r in ranks:
                s.send(msg, copy=copy)

    def broadcast_control(self, cmd: tuple):
        body = pickle.dumps(cmd, protocol=pickle.HIGHEST_PROTOCOL)
        if self.ring_w is not None:
            self.ring_w.send(body, 1)
            return
        for s in self.batch_out:
            s.send(b"C" + body)

    def recv_batch(self, timeout_ms: int = 0):
        """-> ("batch", BatchArrays) | ("control", cmd) | None"""
        if self.ring_r is not None:
            got = self.ring_r.recv()
            if got is None and timeout_ms > 0:
                deadline = time.monotonic() + timeout_ms / 1e3
                while got is None and time.monotonic() < deadline:
                    time.sleep(0.00005)
                    got = self.ring_r.recv()
            if got is None:
                return None
            kind, payload = got
            return ("control", pickle.loads(payload)) if kind == 1 else ("batch", self._decode_batch(memoryview(payload)))
        if self.batch_in is None or not self.batch_in.poll(timeout=timeout_ms):
            return None
        buf = self.batch_in.recv(copy=False).buffer
        if bytes(buf[:1]) == b"C":
            return "control", pickle.loads(buf[1:])
        return "batch", self._decode_batch(buf[1:])

    # output rank -> driver -----------------------------------------------------------------------
    def send_tokens(self, batch_id: int, tokens: List[int], logprobs: Optional[list] = None,
                    prompt_logprobs: Optional[list] = None):
        """`logprobs`: None, or one entry per token (see StepResult.logprobs_list); `prompt_logprobs`: None, or one
        entry per prompt row (see StepResult.prompt_logprobs_list)."""
        self.tok_out.send(pickle.dumps((batch_id, tokens, logprobs, prompt_logprobs),
                                       protocol=pickle.HIGHEST_PROTOCOL))

    def recv_tokens(self):
        out = []
        while self.tok_in is not None and self.tok_in.poll(timeout=0):
            out.append(pickle.loads(self.tok_in.recv()))
        return out

    def close(self, unlink_all: bool = False):
        """Close every socket. `unlink_all` (front-end, after the workers are gone) also removes the ipc socket
        files of the whole engine instance: a worker that was terminated never gets to unlink its own."""
        for s in [self.sock_fe_in, self.sock_fe_out, self.batch_in, self.tok_in, self.tok_out, *self.batch_out]:
            if s is not None:
                s.close(0)
        self.sock_fe_in = self.sock_fe_out = self.batch_in = self.tok_in = self.tok_out = None
        self.batch_out = []
        if self.ring_w is not None:
            self.ring_w.close(unlink=True)
        if self.ring_r is not None:
            self.ring_r.close()
        self.ring_w = self.ring_r = None
        if self.tcp_host is None and self.base.startswith("ipc://"):
            import glob
            root = self.base[len("ipc://"):]
            if unlink_all:
                paths = glob.glob(root + "_*")
            elif self.frontend:
                paths = [f"{root}_fe_out_0"]
            elif self.rank == 0:
                paths = [f"{root}_fe_req_0", f"{root}_tok_0"]
            else:
                paths = [f"{root}_batch_{self.rank}"]          # the endpoints this process bound
            for path in paths:
                try:
                    os.unlink(path)
                except OSError:
                    pass
