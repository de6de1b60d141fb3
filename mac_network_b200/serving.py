"""Host-buffer front end of the inference path: what a caller with numpy / pinned-host batches uses.

The reference feeds each batch from host memory through feed_dict (model.py:1001-1049: createFeedDict); here a batch
goes   host fp32 -> [host cast of the knowledge base to bf16, bf16 path only] -> pinned staging -> H2D on the slot's
stream -> the captured netLength unroll -> D2H of the final state and the attention maps into pinned host memory.
`slots` batches are in flight at once, each on its own CUDA stream, so the PCIe copies of one batch overlap the kernels
of the others.  The knowledge base is 83 % of a batch's bytes; the bf16 read unit only ever reads its bf16 copy
(mac_cast_bf16 would make it on the device), so casting on the host (mac_host_cast_bf16, a thread pool inside the
C library; same bits) halves the H2D traffic -- PCIe, not the GPU, bounds this path.
"""
import ctypes
import os
import torch

from . import _lib
from .mac_cell import MACCell, mac_network


def usable_cpus():
    """CPUs this process may use: affinity mask capped by the cgroup quota (containers)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except Exception:
        pass
    return max(1, n)


def _parse_cpulist(text):
    cpus = set()
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.update(range(int(a), int(b) + 1))
        else:
            cpus.add(int(part))
    return cpus


def gpu_numa_nodes():
    """[NUMA node of visible CUDA device i] (-1 where /sys does not say)."""
    out = []
    for i in range(torch.cuda.device_count()):
        node = -1
        try:
            prop = torch.cuda.get_device_properties(i)
            bus = "%04x:%02x:%02x.0" % (getattr(prop, "pci_domain_id", 0), prop.pci_bus_id, prop.pci_device_id)
            with open("/sys/bus/pci/devices/%s/numa_node" % bus) as f:
                node = int(f.read().strip())
        except Exception:           # noqa: BLE001 -- advisory only
            node = -1
        out.append(node)
    return out


def spread_order(nodes):
    """Visible devices re-ordered round-robin over their NUMA nodes (node order = first appearance, device order kept
    inside a node): [0,0,0,0,1,1,1,1] -> [0,4,1,5,2,6,3,7].  A job of fewer ranks than GPUs then puts its ranks on as many
    sockets as possible, so that each rank's host staging has a socket's memory bandwidth and cores to itself."""
    groups, seen = {}, []
    for i, n in enumerate(nodes):
        if n not in groups:
            groups[n] = []
            seen.append(n)
        groups[n].append(i)
    order, k = [], 0
    while len(order) < len(nodes):
        for n in seen:
            if k < len(groups[n]):
                order.append(groups[n][k])
        k += 1
    return order


def device_for_rank(local_rank, local_world):
    """CUDA device index of a local rank: the identity when every visible GPU is used (or the topology is unknown), else the
    NUMA-spread order above.  Deterministic, so every rank computes the same assignment without talking."""
    n = torch.cuda.device_count()
    if local_world >= n or os.environ.get("MAC_NO_GPU_SPREAD", "0") == "1":
        return local_rank
    nodes = gpu_numa_nodes()
    if len(set(nodes)) <= 1 or any(x < 0 for x in nodes):
        return local_rank
    return spread_order(nodes)[local_rank]


def bind_to_gpu_numa(device_index):
    """Pin this process (and the threads / pinned host buffers it creates afterwards: first touch) to the NUMA node the
    GPU's PCIe root hangs off.  One process per GPU on a 2-socket host otherwise leaves half of the ranks staging their
    batches through the remote socket (SCALE_r01: end-to-end efficiency 0.38 at 8 GPUs with GPUs 4-7 on node 1).
    Returns a description dict; never raises (a container without /sys access simply stays unbound)."""
    info = {"bound": False}
    try:
        prop = torch.cuda.get_device_properties(device_index)
        bus = "%04x:%02x:%02x.0" % (getattr(prop, "pci_domain_id", 0), prop.pci_bus_id, prop.pci_device_id)
        with open("/sys/bus/pci/devices/%s/numa_node" % bus) as f:
            node = int(f.read().strip())
        info.update(pci=bus, numa_node=node)
        if node < 0:
            return info
        with open("/sys/devices/system/node/node%d/cpulist" % node) as f:
            node_cpus = _parse_cpulist(f.read())
        mine = set(os.sched_getaffinity(0))
        target = sorted(node_cpus & mine)
        if not target:
            return info
        os.sched_setaffinity(0, target)
        info.update(bound=True, cpus=len(target))
    except Exception as exc:           # noqa: BLE001 -- advisory only
        info["error"] = repr(exc)[:120]
    return info


class _Slot(object):
    def __init__(self, cfg, params, shape, prec, host_kb_bf16, use_graph, fold_y=None, small_tc=None):
        B, S, N, d, L = shape
        dev = torch.device("cuda", torch.cuda.current_device())
        self.stream = torch.cuda.Stream()
        self.x = {
            "vecQuestions": torch.zeros(B, d, device=dev),
            "questionCntxWords": torch.zeros(B, S, d, device=dev),
            "questionLengths": torch.full((B,), S, dtype=torch.int32, device=dev),
            "knowledgeBase": torch.zeros(B, N, d, device=dev, dtype=torch.bfloat16 if host_kb_bf16 else torch.float32),
        }
        x = self.x
        # questionWords is unused with controlContextual (mac_cell.py:570); the cell takes the contextual words for both
        self.cell = MACCell(x["vecQuestions"], x["questionCntxWords"], x["questionCntxWords"], x["questionLengths"],
                            x["knowledgeBase"], 1.0, 1.0, 1.0, B, False, config=cfg, params=params, prec=prec, fold_y=fold_y,
                            small_tc=small_tc)
        self.L = L
        self.graph = None
        with torch.cuda.stream(self.stream):
            mac_network(self.cell, L)                      # warm-up: packed weights, folded weights, attributes
            self.stream.synchronize()
            if use_graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.stream):
                    mac_network(self.cell, L)
                self.graph = g
        c = self.cell
        self.outs_dev = {"control": c._hc[L], "memory": c._hm[L], "att_kb": c._att_kb, "att_question": c._att_q}
        self.outs_host = {k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in self.outs_dev.items()}
        self.kb_stage = None        # assigned per submit from HostPipeline's small staging ring
        self.h2d_done = torch.cuda.Event()
        self.done = torch.cuda.Event()
        self.busy = False


class HostPipeline(object):
    """`submit(batch)` takes one batch of HOST tensors (fp32; pinned for asynchronous copies) with the keys
    vecQuestions [B,d], questionCntxWords [B,S,d], questionLengths [B] (int32) and knowledgeBase [B,N,d]; it returns a
    ticket.  `result(ticket)` blocks until that batch is done and returns pinned host tensors (final control / memory
    state, per-step KB and question attention maps) that stay valid until the slot is reused `slots` submits later."""

    def __init__(self, cfg, params, shape, prec="bf16", slots=4, use_graph=True, cast_threads=None, fold_y=None,
                 host_cast=None, stage_ring=None):
        """`host_cast`: None = decide here (bf16 path: cast the knowledge base to bf16 on the host if that is faster than the
        PCIe time it saves); False = never.  Callers that run several ranks per socket pass False: the cast makes a pass touch
        ~57 MB of host DRAM (fp32 read + bf16 write + DMA read) instead of 31 MB, and the ranks of one socket share its memory
        bandwidth."""
        self.lib = _lib.load()
        self.shape = shape
        self.prec = prec
        self.host_kb_bf16 = (prec == "bf16" and os.environ.get("MAC_NO_HOST_CAST", "0") != "1"
                             and os.environ.get("MAC_NO_READ_HOIST", "0") != "1" and cfg.is_fast_path
                             and not cfg.unsharedCells and host_cast is not False)
        self.cast_threads = int(cast_threads) if cast_threads else max(1, min(12, usable_cpus() - 2))
        if os.environ.get("MAC_HOST_CAST_THREADS"):
            self.cast_threads = max(1, int(os.environ["MAC_HOST_CAST_THREADS"]))
        self.cast_ms = None
        if self.host_kb_bf16 and os.environ.get("MAC_NO_HOST_CAST", "") != "0":
            # the cast pays off only if it is faster than the PCIe time of the bytes it saves (2 B per KB element at a
            # conservative 25 GB/s); with few host threads per rank (torchrun on a small CPU quota) it is not
            self.cast_ms = self._time_cast(shape)
            saved_ms = shape[0] * shape[2] * shape[3] * 2 / 25e9 * 1e3
            if self.cast_ms > 0.8 * saved_ms:
                self.host_kb_bf16 = False
        if fold_y is None:
            fold_y = slots < 4          # several batches in flight: the unfolded write + projY GEMMs pack better (mac_cell.py)
        # several batches in flight: the tensor-core form of the batch-sized projections (see MACCell.__init__)
        self.slots = [_Slot(cfg, params, shape, prec, self.host_kb_bf16, use_graph, fold_y, small_tc=(slots >= 2))
                      for _ in range(max(1, slots))]
        self._cast_for = None
        self._next = 0
        B, S, N, d, L = shape
        # bf16 staging of the knowledge base through a SMALL ring of pinned buffers (not one buffer per device slot), so that
        # what the cast writes and the H2D engine reads stays in the socket's last-level cache -- the cast then costs DRAM only
        # its fp32 read.  Measured with two ranks on one socket (reasoning-steps/s, both ranks): 30.3k with 12 full-size buffers
        # per rank, 36.9k with 3, 43.4k with 2; no cast: 40.0k.  One rank: 28.4k / 28.9k / 25.2k with 2 / 3 / 12.
        # The batch can also go through the ring in several pieces (MAC_HOST_CAST_CHUNKS), the cast of piece c+1 under the
        # copy of piece c: measured WORSE (4 pieces: 18.6k with one rank, 18.8-24.3k with two) -- every piece is one more
        # wake-up of the cast pool and one more blocking wait in the submit loop -- so the default is one piece.
        self.chunks = max(1, int(os.environ.get("MAC_HOST_CAST_CHUNKS", "1")))
        n_kb = B * N * d
        while n_kb % (self.chunks * 64):
            self.chunks -= 1
        self.chunk_elems = n_kb // self.chunks
        # `stage_ring`: 3 full-size buffers when this rank has its socket to itself (one more pass of slack between a buffer's
        # copy and its next cast), 2 when the socket's cache is shared with another rank's ring (callers pass it; default 3)
        ring = int(os.environ.get("MAC_HOST_STAGE_RING", "0")) or (int(stage_ring) if stage_ring else 3) * self.chunks
        ring = max(2, ring)
        self._stages = ([torch.empty(self.chunk_elems, dtype=torch.bfloat16).pin_memory() for _ in range(ring)]
                        if self.host_kb_bf16 else [])
        self._stage_busy = [None] * len(self._stages)      # event after the copy that last read each buffer
        self._piece = 0                                     # running index of the next piece to cast (pass * chunks + c)
        kb_bytes = B * N * d * (2 if self.host_kb_bf16 else 4)
        self.h2d_bytes = kb_bytes + B * S * d * 4 + B * d * 4 + B * 4
        self.d2h_bytes = sum(v.numel() * v.element_size() for v in self.slots[0].outs_host.values())

    def _time_cast(self, shape):
        import time
        n = shape[0] * shape[2] * shape[3]
        src = torch.zeros(n, dtype=torch.float32).pin_memory()
        dst = torch.empty(n, dtype=torch.bfloat16).pin_memory()
        best = float("inf")
        for _ in range(4):
            t0 = time.perf_counter()
            self.lib.mac_host_cast_bf16(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), n, self.cast_threads)
            best = min(best, time.perf_counter() - t0)
        return best * 1e3

    # -- host cast of the knowledge base on the library's thread pool, one PIECE ahead of the copies
    #    (mac_host_cast_bf16_begin returns at once; no Python threads, so no GIL hand-offs in the submit loop)
    def _cast_begin(self, kb, c):
        """Start the cast of piece c of `kb` into the next staging buffer; returns that buffer's ring index."""
        si = self._piece % len(self._stages)
        self._piece += 1
        if self._stage_busy[si] is not None:
            self._stage_busy[si].synchronize()         # the previous copy out of this staging buffer has finished
            self._stage_busy[si] = None
        src = kb.data_ptr() + 4 * c * self.chunk_elems
        st = self.lib.mac_host_cast_bf16_begin(ctypes.c_void_p(src), ctypes.c_void_p(self._stages[si].data_ptr()),
                                               self.chunk_elems, self.cast_threads)
        if st != 0:
            raise _lib.MacB200Error("mac_host_cast_bf16_begin failed: %d" % st)
        return si

    def prefetch(self, batch):
        """Optional: start the host cast (of the first piece) for the batch that the NEXT submit() will take."""
        if not self.host_kb_bf16:
            return
        kb = batch["knowledgeBase"]
        if self._cast_for is not None:
            if self._cast_for[0] == self._next and self._cast_for[1] is kb:
                return
            self.lib.mac_host_cast_bf16_end()
            self._piece -= 1                           # that piece is discarded: its staging buffer is taken again
        si = self._cast_begin(kb, 0)
        self._cast_for = (self._next, kb, si)

    def submit(self, batch, next_batch=None):
        t = self._next
        slot = self.slots[t % len(self.slots)]
        if self.host_kb_bf16:
            self.prefetch(batch)                       # no-op when the caller (or the previous submit) already started it
            si = self._cast_for[2]
            self._cast_for = None
        self._next = t + 1
        with torch.cuda.stream(slot.stream):
            slot.x["vecQuestions"].copy_(batch["vecQuestions"], non_blocking=True)
            slot.x["questionCntxWords"].copy_(batch["questionCntxWords"], non_blocking=True)
            slot.x["questionLengths"].copy_(batch["questionLengths"], non_blocking=True)
            if self.host_kb_bf16:
                kb, dev = batch["knowledgeBase"], slot.x["knowledgeBase"].view(-1)
                for c in range(self.chunks):
                    self.lib.mac_host_cast_bf16_end()                  # piece c is in its staging buffer
                    cur = si
                    if c + 1 < self.chunks:
                        si = self._cast_begin(kb, c + 1)               # cast of the next piece runs under this piece's copy
                    elif next_batch is not None:
                        si = self._cast_begin(next_batch["knowledgeBase"], 0)
                        self._cast_for = (self._next, next_batch["knowledgeBase"], si)
                    dev[c * self.chunk_elems:(c + 1) * self.chunk_elems].copy_(self._stages[cur], non_blocking=True)
                    ev = torch.cuda.Event()
                    ev.record(slot.stream)
                    self._stage_busy[cur] = ev
            else:
                slot.x["knowledgeBase"].copy_(batch["knowledgeBase"], non_blocking=True)
                if next_batch is not None:
                    self.prefetch(next_batch)
            if slot.graph is not None:
                slot.graph.replay()
            else:
                mac_network(slot.cell, slot.L)
            for k, src in slot.outs_dev.items():
                slot.outs_host[k].copy_(src, non_blocking=True)
            slot.done.record(slot.stream)
        slot.busy = True
        return t

    def result(self, ticket):
        slot = self.slots[ticket % len(self.slots)]
        slot.done.synchronize()
        return slot.outs_host

    def drain(self):
        for s in self.slots:
            if s.busy:
                s.done.synchronize()

    def after(self, stream):
        """Make every slot's stream wait for what has been enqueued on `stream` so far (device-side fork)."""
        ev = torch.cuda.Event()
        ev.record(stream)
        for s in self.slots:
            s.stream.wait_event(ev)

    def wait_streams(self, stream):
        """Make `stream` wait for everything submitted so far (device-side join, for event timing)."""
        for s in self.slots:
            if s.busy:
                stream.wait_event(s.done)
