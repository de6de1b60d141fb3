"""Host-buffer front end of the inference path: what a caller with numpy / pinned-host batches uses.

The reference feeds each batch from host memory through feed_dict (model.py:1001-1049: createFeedDict); here a batch
goes   host fp32 -> [host cast of the knowledge base to bf16, bf16 path only] -> pinned staging -> H2D on the slot's
stream -> the captured netLength unroll -> D2H of the final state and the attention maps into pinned host memory.
`slots` batches are in flight at once, each on its own CUDA stream, so the PCIe copies of one batch overlap the kernels
of the others.  The knowledge base is 83 % of a batch's bytes; the bf16 read unit only ever reads its bf16 copy
(mac_cast_bf16 would make it on the device), so casting on the host (mac_host_cast_bf16, a thread pool inside the
C library; same bits) halves the H2D traffic -- PCIe, not the GPU, bounds this path.

`HostPipeline` is that path for the cell alone (its inputs are the encoder's and the stem's outputs); `ModelPipeline` is the
same scheme for the whole model: question ids and channel-major image features in, answers and attention maps out.
`TrainPipeline` trains the whole model from host batches: the next batch is staged and copied under the current step.
"""
import collections
import ctypes
import os

import numpy as np
import torch

from . import _lib
from ._lib import check, ptr, stream_ptr
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
    if local_world >= n:
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


def _pinned(numel, dtype):
    return torch.empty(numel, dtype=dtype).pin_memory()


def _time_cast(lib, n, threads):
    """Best of four host casts of n fp32 elements to bf16 on the library's pool, in ms."""
    import time
    src = _pinned(n, torch.float32).zero_()
    dst = _pinned(n, torch.bfloat16)
    best = float("inf")
    for _ in range(4):
        t0 = time.perf_counter()
        lib.mac_host_cast_bf16(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(dst.data_ptr()), n, threads)
        best = min(best, time.perf_counter() - t0)
    return best * 1e3


def _cast_pays(cast_ms, numel):
    """The host cast pays off only if it is faster than the PCIe time of the bytes it saves (2 B per element at a
    conservative 25 GB/s); with few host threads per rank (torchrun on a small CPU quota) it is not."""
    return cast_ms <= 0.8 * (numel * 2 / 25e9 * 1e3)


class _CastRing(object):
    """Host cast of one fp32 tensor per batch to bf16 on the library's thread pool (mac_host_cast_bf16_begin returns at once;
    no Python threads, so no GIL hand-offs in the submit loop), one batch ahead of the copies, through a SMALL ring of
    pinned staging buffers (not one buffer per device slot), so that what the cast writes and the H2D engine reads stays in
    the socket's last-level cache -- the cast then costs DRAM only its fp32 read."""

    def __init__(self, lib, numel, ring, threads):
        self.lib, self.threads = lib, threads
        self.stages = [_pinned(numel, torch.bfloat16) for _ in range(ring)]
        self.busy = [None] * ring           # event after the copy that last read each buffer
        self.casts = 0                      # casts started so far: the next one's place in the ring
        self.pending = None                 # (ticket, source tensor, ring index) of the cast in flight

    def begin(self, src):
        """Start the cast of `src` (at most a staging buffer's elements) into the front of the next staging buffer; returns
        that buffer's ring index."""
        si = self.casts % len(self.stages)
        self.casts += 1
        if self.busy[si] is not None:
            self.busy[si].synchronize()              # the previous copy out of this staging buffer has finished
            self.busy[si] = None
        st = self.lib.mac_host_cast_bf16_begin(ctypes.c_void_p(src.data_ptr()), ctypes.c_void_p(self.stages[si].data_ptr()),
                                               min(src.numel(), self.stages[si].numel()), self.threads)
        if st != 0:
            raise _lib.MacB200Error("mac_host_cast_bf16_begin failed: %d" % st)
        return si

    def prefetch(self, ticket, src):
        """Start the cast of `src` for the submit that will carry `ticket`, unless it is the one already in flight."""
        if self.pending is not None:
            if self.pending[0] == ticket and self.pending[1] is src:
                return
            self.lib.mac_host_cast_bf16_end()
            self.casts -= 1                          # that cast is discarded: its staging buffer is taken again
        self.pending = (ticket, src, self.begin(src))

    def take(self, ticket, src):
        """Ring index of the staging buffer that holds (or is receiving) bf16(src); `end()` before copying out of it."""
        self.prefetch(ticket, src)                   # no-op when the caller (or the previous submit) already started it
        si = self.pending[2]
        self.pending = None
        return si

    def end(self):
        self.lib.mac_host_cast_bf16_end()

    def copied(self, si, stream):
        """Call after enqueueing the copy out of staging buffer `si` on `stream`."""
        ev = torch.cuda.Event()
        ev.record(stream)
        self.busy[si] = ev


class _Slot(object):
    """One batch in flight through the cell: its own stream, persistent device inputs, a cell over them, the netLength
    unroll captured as one CUDA graph, pinned host outputs."""

    def __init__(self, cfg, params, shape, prec, host_kb_bf16, use_graph, fold_y=None, small_tc=None):
        B, S, N, d, L = shape
        dev = params.device
        self.stream = torch.cuda.Stream()
        self.x = {
            "vecQuestions": torch.zeros(B, d, device=dev),
            "questionCntxWords": torch.zeros(B, S, d, device=dev),
            "questionLengths": torch.full((B,), S, dtype=torch.int32, device=dev),
            "knowledgeBase": torch.zeros(B, N, d, device=dev, dtype=torch.bfloat16 if host_kb_bf16 else torch.float32),
        }
        self.B, self.L, self.use_graph = B, L, use_graph
        self._cell_kw = dict(config=cfg, params=params, prec=prec, fold_y=fold_y, small_tc=small_tc)
        self.cell = None
        self.graph = None
        self.outs_host = None
        self.kb_stage = None        # assigned per submit from HostPipeline's small staging ring
        self.h2d_done = torch.cuda.Event()
        self.done = torch.cuda.Event()
        self.busy = False
        self.capture()

    def capture(self):
        """A new cell over the slot's inputs, one eager pass (weight packs, folded weights and the scalar biases the kernels
        take as arguments, all of the current parameter version, are built outside the graph), then the capture.  The
        slot's stream first waits for the caller's current stream: whatever wrote the parameters there (an optimizer step, a
        checkpoint restore) is enqueued, not necessarily done, and so are the zeroed workspaces of the new cell."""
        self.graph = None                   # a previous capture's memory goes back before the new one takes its own
        x = self.x
        # questionWords is unused with controlContextual (mac_cell.py:570); the cell takes the contextual words for both
        self.cell = MACCell(x["vecQuestions"], x["questionCntxWords"], x["questionCntxWords"], x["questionLengths"],
                            x["knowledgeBase"], 1.0, 1.0, 1.0, self.B, False, **self._cell_kw)
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            mac_network(self.cell, self.L)                 # warm-up: packed weights, folded weights, attributes
            self.stream.synchronize()
            if self.use_graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.stream):
                    mac_network(self.cell, self.L)
                self.graph = g
        c, L = self.cell, self.L
        self.outs_dev = {"control": c._hc[L], "memory": c._hm[L], "att_kb": c._att_kb, "att_question": c._att_q}
        if self.outs_host is None:          # the shapes do not change with the weights
            self.outs_host = {k: _pinned(v.numel(), v.dtype).view(v.shape) for k, v in self.outs_dev.items()}


class HostPipeline(object):
    """`submit(batch)` takes one batch of HOST tensors (fp32; pinned for asynchronous copies) with the keys
    vecQuestions [B,d], questionCntxWords [B,S,d], questionLengths [B] (int32) and knowledgeBase [B,N,d]; it returns a
    ticket.  `result(ticket)` blocks until that batch is done and returns pinned host tensors (final control / memory
    state, per-step KB and question attention maps) that stay valid until the slot is reused `slots` submits later.

    When the parameter values move (`params.version`: optimizer step, checkpoint restore), the packed weights and the scalar
    biases a captured graph holds by value are stale: the next `submit` drains the pipeline and gives every slot a new cell,
    eager pass and capture before it takes the batch, as `ModelPipeline` does.  `drain()` before writing the parameters."""

    def __init__(self, cfg, params, shape, prec="bf16", slots=4, use_graph=True, cast_threads=None, fold_y=None,
                 host_cast=None, stage_ring=None):
        """`host_cast` (bf16 and fp8 paths, which read only the bf16 knowledge base): None = decide here (cast the knowledge
        base to bf16 on the host if that is faster than the PCIe time it saves); False = never; True = always.  Callers that
        run several ranks per socket pass False: the cast makes a pass touch ~57 MB of host DRAM (fp32 read + bf16 write +
        DMA read) instead of 31 MB, and the ranks of one socket share its memory bandwidth."""
        self.lib = _lib.load()
        self.shape = shape
        self.prec = prec
        self.host_kb_bf16 = (prec in ("bf16", "fp8") and cfg.is_fast_path and not cfg.unsharedCells and host_cast is not False)
        self.cast_threads = int(cast_threads) if cast_threads else max(1, min(12, usable_cpus() - 2))
        self.cast_ms = None
        if self.host_kb_bf16 and host_cast is None:
            self.cast_ms = _time_cast(self.lib, shape[0] * shape[2] * shape[3], self.cast_threads)
            self.host_kb_bf16 = _cast_pays(self.cast_ms, shape[0] * shape[2] * shape[3])
        if fold_y is None:
            fold_y = slots < 4          # several batches in flight: the unfolded write + projY GEMMs pack better (mac_cell.py)
        self.params = params
        self._version = params.version
        # several batches in flight: the tensor-core form of the batch-sized projections (see MACCell.__init__)
        self.slots = [_Slot(cfg, params, shape, prec, self.host_kb_bf16, use_graph, fold_y, small_tc=(slots >= 2))
                      for _ in range(max(1, slots))]
        self._next = 0
        B, S, N, d, L = shape
        # bf16 staging of the knowledge base through _CastRing's small ring of pinned buffers.  Measured with two ranks on one
        # socket (reasoning-steps/s, both ranks): 30.3k with 12 full-size buffers per rank, 36.9k with 3, 43.4k with 2; no
        # cast: 40.0k.  One rank: 28.4k / 28.9k / 25.2k with 2 / 3 / 12.
        # Each buffer takes a whole knowledge base: casting it in several pieces, the cast of piece c+1 under the copy of
        # piece c, measured WORSE (4 pieces: 18.6k with one rank, 18.8-24.3k with two) -- every piece is one more wake-up of
        # the cast pool and one more blocking wait in the submit loop.
        # `stage_ring`: 3 full-size buffers when this rank has its socket to itself (one more pass of slack between a buffer's
        # copy and its next cast), 2 when the socket's cache is shared with another rank's ring (callers pass it; default 3)
        ring = max(2, int(stage_ring) if stage_ring else 3)
        self._ring = _CastRing(self.lib, B * N * d, ring, self.cast_threads) if self.host_kb_bf16 else None
        self._stages = self._ring.stages if self._ring else []
        kb_bytes = B * N * d * (2 if self.host_kb_bf16 else 4)
        self.h2d_bytes = kb_bytes + B * S * d * 4 + B * d * 4 + B * 4
        self.d2h_bytes = sum(v.numel() * v.element_size() for v in self.slots[0].outs_host.values())

    def prefetch(self, batch):
        """Optional: start the host cast for the batch that the NEXT submit() will take."""
        if self.host_kb_bf16:
            self._ring.prefetch(self._next, batch["knowledgeBase"])

    def submit(self, batch, next_batch=None):
        if self.params.version != self._version:
            self.drain()
            for s in self.slots:
                s.capture()
            self._version = self.params.version
        t = self._next
        slot = self.slots[t % len(self.slots)]
        if self.host_kb_bf16:
            si = self._ring.take(t, batch["knowledgeBase"])
        self._next = t + 1
        with torch.cuda.stream(slot.stream):
            slot.x["vecQuestions"].copy_(batch["vecQuestions"], non_blocking=True)
            slot.x["questionCntxWords"].copy_(batch["questionCntxWords"], non_blocking=True)
            slot.x["questionLengths"].copy_(batch["questionLengths"], non_blocking=True)
            if self.host_kb_bf16:
                self._ring.end()                                       # the knowledge base is in its staging buffer
                if next_batch is not None:                             # the next batch's cast runs under this copy
                    self._ring.prefetch(self._next, next_batch["knowledgeBase"])
                slot.x["knowledgeBase"].view(-1).copy_(self._stages[si], non_blocking=True)
                self._ring.copied(si, slot.stream)
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


def _check_image_dtype(image_dtype):
    """The pipelines' `image_dtype`: the stored format of the features, fp32 (the default) or fp16."""
    if image_dtype not in (torch.float32, torch.float16):
        raise ValueError("image_dtype must be torch.float32 or torch.float16, got %r" % (image_dtype,))


def _check_f16(v, what):
    """An fp16 pipeline takes fp16 features only: rounding fp32 ones here would change the model's input silently."""
    if v.dtype != torch.float16:
        raise ValueError("%s must be fp16 with image_dtype=torch.float16, got %s" % (what, v.dtype))


class _ModelSlot(object):
    """One batch in flight through the whole model: its own stream, persistent device inputs, its own evaluation-mode
    encoder / stem / cell / output unit over the model's parameter tensors, the forward captured as one CUDA graph, pinned
    host outputs."""

    def __init__(self, model, shape, image_dtype, use_graph, topk, images=None):
        B, S, H, W = shape
        t, cfg = model.trainer, model.cfg
        p = t.params
        self.model, self.B, self.topk, self.use_graph = model, B, topk, use_graph
        C = model._stem.in_dim
        self.stream = torch.cuda.Stream()
        self.x = {"questions": torch.zeros(B, S, dtype=torch.int32, device=p.device),
                  "questionLengths": torch.full((B,), S, dtype=torch.int32, device=p.device),
                  "images": torch.zeros(B if images is None else images, C, H, W, device=p.device, dtype=image_dtype)}
        self.x.update(self._index_inputs(B, images, p.device))
        from .encoder import QuestionEncoder
        from .output_unit import OutputUnit
        from .stem import Stem
        version = lambda: p.version
        self.enc = QuestionEncoder({k: p.t[k] for k in t._enc_specs}, keep_input=1.0, keep_question=1.0,
                                   prec=model._enc.prec, version=version)
        self.stem = Stem({k: p.t[k] for k in t._stem_specs}, relu=cfg.relu, prec=model._stem.prec, version=version,
                         strides=model._stem.strides, linear=model._stem.linear, location=model._stem.location)
        self.out = OutputUnit({k: p.t[k] for k in p.specs if k.startswith(("outputUnit/", "classifier/"))}, relu=cfg.relu,
                              keep=1.0, version=version, bn_decay=cfg.bnDecay, **t.out.options)
        self.cell = None
        self.graph = None
        self.outs_host = None
        self.done = torch.cuda.Event()
        self.busy = False
        self.capture()

    def _index_inputs(self, B, images, device):
        """The graph's device index inputs: with images=U, question b reads image imageIndex[b] of the U the stem runs over."""
        return {} if images is None else {"imageIndex": torch.zeros(B, dtype=torch.int32, device=device)}

    def _forward(self):
        x = self.x
        words, cntx, vecq = self.enc.forward(x["questions"], x["questionLengths"])
        kb = self.stem.forward_nchw(x["images"])
        return self._answer(vecq, words, cntx, kb, x.get("imageIndex"))

    def _answer(self, vecq, words, cntx, kb, idx):
        """The cell over the knowledge base `kb` (gathered by `idx` when given), the output unit and the top-k: the outputs
        of one pass."""
        from .output_unit import answer_topk
        m = self.model
        if self.cell is None:       # MACCell's own errors (flag set / precision outside its inference forms) pass through
            self.cell = MACCell(vecq, words, cntx, self.x["questionLengths"], kb, 1.0, 1.0, 1.0, self.B, False, config=m.cfg,
                                params=m.trainer.params, prec=m.prec, kbIndex=idx)
        else:
            self.cell.rebind(vecq, words, cntx, kb, kbIndex=idx)
        c = self.cell
        _, memory = mac_network(c, m.L)
        logits = self.out.logits(memory, vecq)
        ids, probs = answer_topk(logits, self.topk)
        outs = {"answers": ids, "probs": probs, "logits": logits, "memory": memory, "att_kb": c._att_kb,
                "att_question": c._att_q}
        if c.attentions["gate"]:
            outs["gate"] = torch.stack(c.attentions["gate"])
        if c.attentions["self"]:            # step i attends over its i + 1 history rows: zero-padded to [L, B, L]
            outs["self"] = torch.zeros(m.L, self.B, m.L, device=memory.device)
            for i, a in enumerate(c.attentions["self"]):
                outs["self"][i, :, :i + 1].copy_(a)
        return outs

    def _host_outputs(self):
        if self.outs_host is None:          # the shapes do not change with the weights
            self.outs_host = {k: _pinned(v.numel(), v.dtype).view(v.shape) for k, v in self.outs_dev.items()}

    def capture(self):
        """One eager pass (weight packs and folded weights of the current parameter version are built outside the graph),
        then the capture.  The outputs of the pass that was captured are the graph's static output tensors.  The slot's
        stream first waits for the caller's current stream: whatever wrote the parameters there (an optimizer step, a
        checkpoint restore) or built packs from them (`runBatch`) is enqueued, not necessarily done."""
        self.graph = None                   # a previous capture's memory goes back before the new one takes its own
        self.cell = None                    # built again by the eager pass below
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            self.outs_dev = self._forward()
            self.stream.synchronize()
            if self.use_graph:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=self.stream):
                    self.outs_dev = self._forward()
                self.graph = g
        self._host_outputs()

    def enqueue(self, questions, lengths, images, copied=None, index=None):
        """H2D copies -> forward -> D2H copies on this slot's stream; returns after enqueueing.  `images` is host memory of
        the slot's image type (the caller's fp32 tensor or a bf16 staging buffer), any shape with the element count of the
        slot's images or, with `index` (the slot's imageIndex), of their first k, or a callable that returns it, called once
        the small copies are enqueued (the host cast is waited for there); `copied(stream)` is called once the image copy is
        enqueued."""
        with torch.cuda.stream(self.stream):
            self.x["questions"].copy_(questions, non_blocking=True)
            self.x["questionLengths"].copy_(lengths, non_blocking=True)
            if index is not None:
                self.x["imageIndex"].copy_(index, non_blocking=True)
            if callable(images):
                images = images()
            self.x["images"].view(-1)[:images.numel()].copy_(images.view(-1), non_blocking=True)
            if copied is not None:
                copied(self.stream)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.outs_dev = self._forward()
            for k, src in self.outs_dev.items():
                self.outs_host[k].copy_(src, non_blocking=True)
            self.done.record(self.stream)
        self.busy = True


class _CachedSlot(_ModelSlot):
    """A `_ModelSlot` that reads its knowledge bases from the pipeline's device pool (`ModelPipeline(cache=C)`), with two
    captured graphs: the stem graph (ingest and stem over the slot's U image rows, then `mac_kb_pool_insert` into the pool
    rows `insertSlot` names) and the cell graph (encoder, then for a bf16 pool `mac_kb_gather_bf16` of the rows `kbSlot`
    names, then the cell -- over the fp32 pool itself with kbIndex = kbSlot otherwise --, the output unit and the top-k)."""

    def __init__(self, model, shape, use_graph, topk, images, pool, image_dtype=torch.float32):
        B = int(shape[0])
        self.pool = pool
        self.lib = _lib.load()
        self.kb16 = (torch.empty((B,) + tuple(pool.shape[1:]), dtype=torch.bfloat16, device=pool.device)
                     if pool.dtype == torch.bfloat16 else None)
        self.stem_graph = None
        self.chunks = -(-B // images)       # stem passes of a batch with B misses
        # insert slots of each stem pass, then the batch's kbSlot: written on the host before any copy out of it is enqueued
        self.index_host = _pinned(self.chunks * images + B, torch.int32)
        self.index_copied = torch.cuda.Event()      # after the last copy out of index_host
        self.index_busy = False
        self.covered = {}       # other slot -> (ticket, stem pass) of its latest work this slot's stream has waited for
        super(_CachedSlot, self).__init__(model, shape, image_dtype, use_graph, topk, images)

    def _index_inputs(self, B, images, device):
        return {"insertSlot": torch.full((images,), -1, dtype=torch.int32, device=device),
                "kbSlot": torch.zeros(B, dtype=torch.int32, device=device)}

    def _stem_pass(self):
        kb = self.stem.forward_nchw(self.x["images"])
        U, N, d = kb.shape
        check(self.lib.mac_kb_pool_insert(ptr(kb), ptr(self.x["insertSlot"]), ptr(self.pool), int(self.kb16 is not None), U,
                                          self.pool.shape[0], N, d, stream_ptr()), "mac_kb_pool_insert")

    def _forward(self):
        x = self.x
        words, cntx, vecq = self.enc.forward(x["questions"], x["questionLengths"])
        if self.kb16 is None:
            return self._answer(vecq, words, cntx, self.pool, x["kbSlot"])
        C, N, d = self.pool.shape
        check(self.lib.mac_kb_gather_bf16(ptr(self.pool), ptr(x["kbSlot"]), ptr(self.kb16), self.B, C, N, d, stream_ptr()),
              "mac_kb_gather_bf16")
        return self._answer(vecq, words, cntx, self.kb16, None)

    def capture(self):
        """As `_ModelSlot.capture`, for both graphs.  The insert slots are set to -1 first, so neither the eager nor the
        captured stem pass writes a pool row."""
        self.graph = self.stem_graph = None
        self.cell = None
        self.stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self.stream):
            self.x["insertSlot"].fill_(-1)
            self._stem_pass()
            self.outs_dev = self._forward()
            self.stream.synchronize()
            if self.use_graph:
                gs, g = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
                with torch.cuda.graph(gs, stream=self.stream):
                    self._stem_pass()
                with torch.cuda.graph(g, stream=self.stream):
                    self.outs_dev = self._forward()
                self.stem_graph, self.graph = gs, g
        self._host_outputs()

    def enqueue_cached(self, questions, lengths, waits, passes, kb_slots, done):
        """Wait for `waits` (events of other slots) -> H2D of the questions -> per stem pass (images [n <= U, C, H, W] host,
        insert slots [U]): its slots and images, the stem graph, an event -> kbSlot -> the cell graph -> D2H -> `done`, a
        fresh event of this batch that becomes the slot's `done`, on this slot's stream.  Returns the events recorded after
        each stem pass."""
        U = self.x["insertSlot"].shape[0]
        h = self.index_host
        if self.index_busy:
            self.index_copied.synchronize()         # the copies out of index_host of this slot's previous batch are done
        for j, (_, slots) in enumerate(passes):
            h[j * U:(j + 1) * U].copy_(torch.from_numpy(slots))
        h[self.chunks * U:].copy_(torch.from_numpy(kb_slots))
        events = []
        with torch.cuda.stream(self.stream):
            for ev in waits:
                self.stream.wait_event(ev)
            self.x["questions"].copy_(questions, non_blocking=True)
            self.x["questionLengths"].copy_(lengths, non_blocking=True)
            for j, (images, _) in enumerate(passes):
                self.x["insertSlot"].copy_(h[j * U:(j + 1) * U], non_blocking=True)
                self.x["images"][:images.shape[0]].copy_(images, non_blocking=True)
                if self.stem_graph is not None:
                    self.stem_graph.replay()
                else:
                    self._stem_pass()
                ev = torch.cuda.Event()
                ev.record(self.stream)
                events.append(ev)
            self.x["kbSlot"].copy_(h[self.chunks * U:], non_blocking=True)
            self.index_copied.record(self.stream)
            self.index_busy = True
            if self.graph is not None:
                self.graph.replay()
            else:
                self.outs_dev = self._forward()
            for k, src in self.outs_dev.items():
                self.outs_host[k].copy_(src, non_blocking=True)
            self.done = done
            self.done.record(self.stream)
        self.busy = True
        return events


_Plan = collections.namedtuple("_Plan", "hits miss rows victims")


class _KBCache(object):
    """Host bookkeeping of `ModelPipeline(cache=C)`'s device pool: which image key each of the C rows holds (`key`, and
    `rows`: key -> row in least-recently-used order), per row the (ticket, stem pass, event) of the stem pass that wrote it
    and, on each of the `slots` streams, the last batch that read it as (ticket, that batch's own done event) -- reads on
    different streams are not ordered, so the last reader alone does not cover the others.  `plan` changes nothing;
    `commit` applies a plan once the batch has been checked."""

    def __init__(self, capacity, slots):
        self.capacity, self.slots = int(capacity), int(slots)
        self.stats = {"hits": 0, "misses": 0, "evictions": 0, "image_bytes": 0}
        self.clear()

    def clear(self):
        self.rows = collections.OrderedDict()       # key -> row, least recently used first
        self.key = [None] * self.capacity
        self.written = [None] * self.capacity       # (ticket, stem pass, event) of the pass that wrote the row
        self.reader = [[None] * self.slots for _ in range(self.capacity)]   # per row and slot: (ticket, done) of a reader
        self.free = list(range(self.capacity))      # rows that hold no key, taken from the front

    def plan(self, keys):
        """`keys`: a batch's distinct image keys in first-occurrence order.  Their rows where held (hits), the missing keys
        in that order, the row each will be written to -- free rows first, then the least recently used rows the batch does
        not read -- and which of those are evictions."""
        hits = [self.rows[k] for k in keys if k in self.rows]
        miss = [k for k in keys if k not in self.rows]
        rows = self.free[:len(miss)]
        victims = []
        if len(rows) < len(miss):
            used = set(hits)
            for r in self.rows.values():
                if r not in used:
                    victims.append(r)
                    if len(rows) + len(victims) == len(miss):
                        break
        return _Plan(hits, miss, rows + victims, victims)

    def commit(self, plan, ticket, done=None):
        """Apply `plan` for the batch `ticket`, whose done event (recorded after its cell pass) is `done`."""
        for r in plan.hits:
            self.rows.move_to_end(self.key[r])
            self.reader[r][ticket % self.slots] = (ticket, done)
        for r in plan.victims:
            del self.rows[self.key[r]]
        del self.free[:len(plan.rows) - len(plan.victims)]
        for k, r in zip(plan.miss, plan.rows):
            self.key[r], self.written[r] = k, None
            self.reader[r] = [None] * self.slots
            self.reader[r][ticket % self.slots] = (ticket, done)
            self.rows[k] = r
        self.stats["hits"] += len(plan.hits)
        self.stats["misses"] += len(plan.miss)
        self.stats["evictions"] += len(plan.victims)


class ModelPipeline(object):
    """The whole model from host buffers: what a caller who has questions and image features -- not the encoder's and the
    stem's outputs `HostPipeline` takes -- uses to ask the model for answers, with no labels.

        pipe = ModelPipeline(model, shape=(B, S, H, W), slots=4)
        t = pipe.submit({"questions": int32 [B, S] (0-padded), "questionLengths": int32 [B], "images": fp32 [B, C, H, W]})
        out = pipe.result(t)          # pinned host tensors, valid until the slot is reused `slots` submits later

    `model` is a `MACnet`: the pipeline serves the weights in `model.trainer.params` with the model's `prec` and evaluation
    stem / encoder precisions (to serve EMA shadows, load them first: `load_checkpoint(use_ema=True)`; `runBatch`'s per-batch
    EMA swap has no counterpart here).  Each of the `slots` batches in flight has its own stream and runs
    `mac_ingest_nchw` -> stem -> encoder -> `mac_network` -> `OutputUnit.logits` -> `mac_answer_topk` as ONE captured CUDA
    graph, so one batch's PCIe copies overlap another's kernels.  Images are 96 % of a batch's bytes; the bf16 stem reads
    only bf16(x), so with it `host_cast` (None: decide by timing, as `HostPipeline` does; True / False: forced) casts them
    on the host and halves the H2D traffic.  With any other stem the features stay fp32.  Measured on an H100 (DESIGN.md
    section 8) the fp32 copies ran at 27-36 GB/s with four slots and the cast, bound by the host's cores, was the slower
    path; callers who see the copies keep up should pass `host_cast=False`.

    `out`: `answers` int32 [B, topk] (column 0 is the prediction), `probs` [B, topk], `logits` [B, A], `memory` [B, d],
    `att_kb` [L, B, Ho*Wo] (the stem's output grid, `Stem.grid`), `att_question` [L, B, S], and `gate` [L, B, d] /
    `self` [L, B, L] (step i's i + 1 weights, zero beyond) when the flag set has them.

    Several questions per image: with `images=U` (1 <= U <= B) a batch carries k <= U distinct images and each question's
    image number,

        pipe = ModelPipeline(model, shape=(B, S, H, W), slots=4, images=8)
        t = pipe.submit({"questions": ..., "questionLengths": ..., "images": fp32 [k, C, H, W], "imageIndex": int32 [B]})

    with 1 <= k <= U and every imageIndex[b] in [0, k).  Only the k images cross PCIe; the captured graph runs the ingest and
    the stem over the slot's U image rows (rows k..U-1 hold a previous batch's data that no question reads) and the cell
    gathers each question's knowledge base from them (`MACCell(kbIndex=)`, `mac_kb_gather`).  The index is a device input
    of the graph like the questions: a new index pattern or a new k needs no new capture.

    Knowledge bases kept on the device across batches: with `cache=C` (C >= B, and `images=U` the number of images one stem
    pass takes) the pipeline keeps the knowledge bases of the last C distinct images it has seen in one device pool
    [C, Ho*Wo, d], shared by all slots, keyed by the caller's integer image ids,

        pipe = ModelPipeline(model, shape=(B, S, H, W), slots=4, images=16, cache=15000)
        t = pipe.submit({"questions": ..., "questionLengths": ..., "imageIds": int [B], "images": load})

    where `load(ids)` is given the batch's ids that are not in the cache (int64 numpy [m], first-occurrence order; called
    only when m > 0) and returns their fp32 features [m, C, H, W], numpy or a host tensor (pinned makes the copy
    asynchronous; a pinned result must not be written until its ticket's result is read).  Per slot there are two captured
    graphs: the stem graph, replayed once per U missing images, runs the ingest and the stem over the slot's U image rows
    and writes them into the pool rows its device input `insertSlot` names (`mac_kb_pool_insert`); the cell graph runs the
    encoder and the cell over the pool rows of `kbSlot` [B].  A batch whose images are all cached copies no image byte and
    launches no ingest or stem kernel.  The pool is bf16 where the cell's read unit reads only bf16 (the bf16 and e4m3
    hoisted forms: the cell graph gathers it with `mac_kb_gather_bf16`) and fp32 otherwise (the cell gathers it itself,
    `MACCell(kbIndex=)`); either way the outputs are bit for bit those of `images=U` without a cache.  When a pool row is
    evicted (least recently used first, never a row the batch reads) the slot's stream first waits for the batches of
    other slots that read it, and a batch that reads a row written by a batch still in flight on another slot waits for that
    write; neither waits on the host.  A key must name one feature map for the cache's lifetime (CLEVR's image_index
    repeats across its splits: one pipeline per image file, or `clear_cache()` between them); a weight update empties the
    cache.  `host_cast` is off with a cache.  `cache_stats()` counts hits, misses, evictions and image bytes copied.

    Features stored in fp16: with `image_dtype=torch.float16` the batch's images (and a cache's loader results) must be
    fp16 host arrays -- anything else raises `ValueError` before anything is staged, so fp32 features are never rounded
    silently.  The slots' pinned staging and the graphs' device image inputs are fp16, half the bytes cross PCIe (counted by
    `h2d_bytes` and `cache_stats()`), and the captured ingest is `mac_ingest_nchw_f16`, which widens on the device: every
    output is bit for bit what the default pipeline computes from the fp32 widening of the same features.  `host_cast=True`
    is refused with it (there is nothing left to cast).  The default, `torch.float32`, widens an fp16 batch on the host.

    Questions are padded with 0 to the pipeline's fixed S (a captured graph cannot trim a batch to its longest question as
    `runBatch` does); the kernels mask by length, so attention at positions >= length is exactly 0.

    When the parameter values move (`params.version`: optimizer step, checkpoint restore), the packed weights are rebuilt as
    new tensors a captured graph would not see: the next `submit` drains the pipeline and captures every slot again before
    it takes the batch.  Each slot's stream waits there for the caller's current stream, so an update enqueued on that
    stream (`DPTrainer`'s optimizer step does not synchronise) is complete before the packs are rebuilt from it.  The
    other direction is the caller's: batches in flight read the parameters, so `drain()` before writing them.

    Memory: every slot has its own encoder and stem and with them its own weight packs (about 14 MB per slot at 1024 -> 512
    -> 512), and its graph's private pool holds its own patch matrices (231 MB for layer 0 at 64x1024x14x14)."""

    def __init__(self, model, shape, slots=4, use_graph=True, topk=1, host_cast=None, cast_threads=None, stage_ring=None,
                 images=None, cache=None, image_dtype=torch.float32):
        B, S, H, W = [int(v) for v in shape]
        _check_image_dtype(image_dtype)
        if image_dtype == torch.float16 and host_cast:
            raise ValueError("host_cast=True casts fp32 features to bf16 on the host: with image_dtype=torch.float16 the "
                             "features cross PCIe as stored and are widened on the device")
        p = model.trainer.params
        C = model._stem.in_dim
        nfc = len([k for k in p.t if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
        A = int(p.t["classifier/linearLayerfc_%d/weights/weight" % (nfc - 1)].shape[1])
        if min(B, S, H, W) <= 0 or slots < 1:
            raise ValueError("shape (B, S, H, W) and slots must be positive, got %r, slots = %r" % (shape, slots))
        if C % 64:
            raise ValueError("the image features have %d channels: mac_ingest_nchw needs a multiple of 64" % C)
        if not 1 <= int(topk) <= min(8, A):
            raise ValueError("topk must be in 1..min(8, %d answers), got %r" % (A, topk))
        if images is not None and not (isinstance(images, int) and 1 <= images <= B):
            raise ValueError("images must be None or an int in 1..B = %d, got %r" % (B, images))
        if cache is not None:
            if images is None:
                raise ValueError("cache=C needs images=U: the number of images one stem pass takes")
            if isinstance(cache, bool) or not isinstance(cache, int) or cache < B:
                raise ValueError("cache must be None or an int >= B = %d (every batch's images must fit), got %r" % (B, cache))
            if model.cfg.memDim % 8:
                raise ValueError("cache=C needs memDim %% 8 == 0 (the pool kernels' 16-byte vectors), got %d" % model.cfg.memDim)
        self.images, self.image_dtype = images, image_dtype
        self.lib = _lib.load()
        self.model, self.params, self.shape, self.C, self.topk = model, p, (B, S, H, W), C, int(topk)
        self.use_graph = bool(use_graph)
        self.cast_threads = int(cast_threads) if cast_threads else max(1, min(12, usable_cpus() - 2))
        numel = (B if images is None else images) * C * H * W
        self.host_cast = (model._stem.prec == "bf16" and host_cast is not False and cache is None
                          and image_dtype == torch.float32)
        self.cast_ms = None
        if self.host_cast and host_cast is None:
            self.cast_ms = _time_cast(self.lib, numel, self.cast_threads)
            self.host_cast = _cast_pays(self.cast_ms, numel)
        self._version = p.version
        self._cache = self.pool = None
        if cache is None:
            slot_dtype = torch.bfloat16 if self.host_cast else image_dtype
            self.slots = [_ModelSlot(model, self.shape, slot_dtype, self.use_graph, self.topk, images)
                          for _ in range(int(slots))]
        else:
            # the pool holds what the cell's read unit reads: bf16 for the bf16 and e4m3 hoisted forms (MACCell's
            # _kb_gather_bf16 condition), the stem's fp32 rows for every other form
            cfg = model.cfg
            pool_bf16 = model.prec in ("bf16", "fp8") and cfg.is_fast_path and not cfg.unsharedCells
            n_kb = int(np.prod(model._stem.grid(H, W)))             # the stem's output grid
            self.pool = torch.zeros(cache, n_kb, cfg.memDim, dtype=torch.bfloat16 if pool_bf16 else torch.float32,
                                    device=p.device)
            self._cache = _KBCache(cache, slots)
            self.slots = [_CachedSlot(model, self.shape, self.use_graph, self.topk, images, self.pool, image_dtype)
                          for _ in range(int(slots))]
        self._ring = (_CastRing(self.lib, numel, max(2, int(stage_ring) if stage_ring else 3), self.cast_threads)
                      if self.host_cast else None)
        self._next = 0
        self._ahead = None                  # (next_batch["images"] as given, its host tensor) of the cast in flight
        # with images=U: a batch of k images copies k of the U counted here; with cache=C only the questions, their lengths
        # and kbSlot are counted (cache_stats() counts the image bytes, and each stem pass adds U * 4 bytes of insert slots)
        self.h2d_bytes = (numel * (2 if self.host_cast or image_dtype == torch.float16 else 4) + B * S * 4 + B * 4
                          + (0 if images is None else B * 4))
        if cache is not None:
            self.h2d_bytes = B * S * 4 + B * 4 + B * 4
        self.d2h_bytes = sum(v.numel() * v.element_size() for v in self.slots[0].outs_host.values())

    def _host(self, batch):
        """The batch's host tensors (questions, lengths, images, and with images=U the image index, else None), checked
        against the pipeline's shape; ValueError before anything is enqueued."""
        B, S, H, W = self.shape
        k = B
        if self.images is None:
            if "imageIndex" in batch:
                raise ValueError("imageIndex is for a pipeline built with images=U")
        else:
            if "imageIndex" not in batch:
                raise ValueError("a pipeline built with images=%d needs the batch's imageIndex" % self.images)
            k = torch.as_tensor(batch["images"]).shape[0]
            if not 1 <= k <= self.images:
                raise ValueError("a batch carries 1..%d images, got %d" % (self.images, k))
        want = (("questions", (B, S), torch.int32), ("questionLengths", (B,), torch.int32),
                ("images", (k, self.C, H, W), torch.float32))
        if self.images is not None:
            want += (("imageIndex", (B,), torch.int32),)
        out = []
        for key, shp, dtype in want:
            v = torch.as_tensor(batch[key])
            if v.device.type != "cpu" or tuple(v.shape) != shp:
                raise ValueError("%s must be a host tensor of shape %s, got %s on %s" % (key, shp, tuple(v.shape), v.device))
            if key == "images" and self.image_dtype == torch.float16:
                _check_f16(v, "the batch's images")
                dtype = torch.float16
            out.append(v.to(dtype).contiguous())
        if self.images is None:
            return out + [None]
        idx = torch.as_tensor(batch["imageIndex"])
        if idx.dtype.is_floating_point or idx.dtype == torch.bool or not bool(((idx >= 0) & (idx < k)).all()):
            raise ValueError("imageIndex must hold integers in [0, %d) (the batch's images)" % k)
        return out

    def submit(self, batch, next_batch=None):
        """Enqueue one batch (numpy arrays or host tensors; pinned memory makes the copies asynchronous) and return its
        ticket.  `next_batch`: the batch the next submit will take, whose host cast then runs under this batch's copies."""
        if self._cache is not None:
            return self._submit_cached(batch)
        q, ql, img, idx = self._host(batch)
        if self._ahead is not None and self._ahead[0] is batch["images"]:
            img = self._ahead[1]                           # the tensor whose cast the previous submit started
        nxt = self._host(next_batch)[2] if (next_batch is not None and self.host_cast) else None
        self._ahead = None if nxt is None else (next_batch["images"], nxt)
        if self.params.version != self._version:
            self.drain()
            for s in self.slots:
                s.capture()
            self._version = self.params.version
        t = self._next
        slot = self.slots[t % len(self.slots)]
        self._next = t + 1
        if not self.host_cast:
            slot.enqueue(q, ql, img, index=idx)
            return t
        si = self._ring.take(t, img)

        def staged():                                      # after the small copies are enqueued, as in HostPipeline.submit
            self._ring.end()                               # the images are in their staging buffer
            if nxt is not None:                            # the next batch's cast runs under this batch's copies
                self._ring.prefetch(self._next, nxt)
            return self._ring.stages[si][:img.numel()]
        slot.enqueue(q, ql, staged, copied=lambda stream: self._ring.copied(si, stream), index=idx)
        return t

    def _checked_ids(self, batch):
        """With cache=C: the batch's questions and lengths as host tensors, its image keys as Python ints and its loader,
        checked against the pipeline's shape; ValueError before anything is enqueued."""
        B, S = self.shape[:2]
        if "imageIndex" in batch:
            raise ValueError("a pipeline built with cache=C takes imageIds and a loader, not imageIndex")
        for key in ("questions", "questionLengths", "imageIds", "images"):
            if key not in batch:
                raise ValueError("the batch has no %s" % key)
        out = []
        for key, shp in (("questions", (B, S)), ("questionLengths", (B,))):
            v = torch.as_tensor(batch[key])
            if v.device.type != "cpu" or tuple(v.shape) != shp:
                raise ValueError("%s must be a host tensor of shape %s, got %s on %s" % (key, shp, tuple(v.shape), v.device))
            out.append(v.to(torch.int32).contiguous())
        ids = torch.as_tensor(batch["imageIds"])
        if (ids.device.type != "cpu" or tuple(ids.shape) != (B,) or ids.dtype.is_floating_point or ids.dtype.is_complex
                or ids.dtype == torch.bool):
            raise ValueError("imageIds must be a host array of %d integers, got %s %s" % (B, ids.dtype, tuple(ids.shape)))
        if not callable(batch["images"]):
            raise ValueError("with cache=C the batch's images are a loader: a callable that takes the missing ids")
        return out + [ids.tolist(), batch["images"]]

    def _loaded(self, load, miss):
        """The loader's features of the missing keys, checked: a host tensor [m, C, H, W] of the pipeline's image dtype."""
        H, W = self.shape[2:]
        res = load(np.asarray(miss, dtype=np.int64))
        name = "fp16" if self.image_dtype == torch.float16 else "fp32"
        try:
            v = torch.as_tensor(res)
        except (TypeError, RuntimeError) as exc:
            raise ValueError("the images loader must return an array of %s features: %s" % (name, exc))
        want = (len(miss), self.C, H, W)
        if v.device.type != "cpu" or v.dtype != self.image_dtype or tuple(v.shape) != want:
            raise ValueError("the images loader must return host %s features of shape %s (NCHW), got %s %s on %s"
                             % (name, want, v.dtype, tuple(v.shape), v.device))
        return v.contiguous()

    def _submit_cached(self, batch):
        q, ql, ids, load = self._checked_ids(batch)
        if self.params.version != self._version:
            self.drain()
            self._cache.clear()
            for s in self.slots:
                s.capture()
            self._version = self.params.version
        cache, U, n = self._cache, self.images, len(self.slots)
        keys = list(dict.fromkeys(ids))                     # distinct keys, first-occurrence order
        plan = cache.plan(keys)
        imgs = self._loaded(load, plan.miss) if plan.miss else None
        # nothing has changed so far; from here on the batch is enqueued
        t = self._next
        si = t % n
        slot = self.slots[si]
        self._next = t + 1
        waits = []
        done = torch.cuda.Event()             # this batch's: recorded after its cell pass, the last read of the pool

        def wait_for(sj, upto, ev):           # make slot si's stream wait for slot sj's work up to (ticket, pass)
            if sj != si and slot.covered.get(sj, (-1, -1)) < upto:
                slot.covered[sj] = upto
                waits.append(ev)
        for r in plan.victims:                # write after read: the row's last reader on every slot has finished
            for sj, reader in enumerate(cache.reader[r]):
                if reader is not None:        # that reader's own done event, not the slot's latest batch
                    wait_for(sj, (reader[0], float("inf")), reader[1])
        for r in plan.hits:                   # read after write: the stem pass that wrote the row has finished
            if cache.written[r] is not None:
                wt, wp, ev = cache.written[r]
                wait_for(wt % n, (wt, wp), ev)
        cache.commit(plan, t, done)
        passes = []
        for j in range(0, len(plan.miss), U):
            slots_j = np.full(U, -1, dtype=np.int32)
            rows_j = plan.rows[j:j + U]
            slots_j[:len(rows_j)] = rows_j
            passes.append((imgs[j:j + U], slots_j))
        kb_slots = np.asarray([cache.rows[k] for k in ids], dtype=np.int32)
        events = slot.enqueue_cached(q, ql, waits, passes, kb_slots, done)
        for j, ev in enumerate(events):
            for r in plan.rows[j * U:(j + 1) * U]:
                cache.written[r] = (t, j, ev)
        cache.stats["image_bytes"] += 0 if imgs is None else imgs.numel() * imgs.element_size()
        return t

    def cache_stats(self):
        """With cache=C: {"hits", "misses"} (distinct images of each batch found in the cache / run through the stem),
        "evictions", "image_bytes" (features copied to the device) since construction, and "resident" (images held now)."""
        if self._cache is None:
            raise ValueError("cache_stats() is for a pipeline built with cache=C")
        return dict(self._cache.stats, resident=len(self._cache.rows))

    def clear_cache(self):
        """With cache=C: wait for the batches in flight, then forget every cached image (the statistics keep counting).
        Use it between image files whose keys overlap."""
        if self._cache is None:
            raise ValueError("clear_cache() is for a pipeline built with cache=C")
        self.drain()
        self._cache.clear()

    def result(self, ticket):
        """Block until the batch of `ticket` is done; its outputs stay valid until `slots` further submits."""
        if not self._next - len(self.slots) <= ticket < self._next:
            raise ValueError("ticket %r is not one of the last %d submits" % (ticket, len(self.slots)))
        slot = self.slots[ticket % len(self.slots)]
        slot.done.synchronize()
        return slot.outs_host

    def predictions(self, out):
        """The answers of a `result` as the model's `answer_decoder` spells them (ids without one)."""
        dec = self.model.decode
        return [dec(int(i)) if dec else int(i) for i in out["answers"][:, 0]]

    def drain(self):
        for s in self.slots:
            if s.busy:
                s.done.synchronize()


class _TrainSlot(object):
    """One training batch in flight: pinned host staging and device inputs, the step's pinned results, and the event of the
    step that reads them."""

    def __init__(self, B, S, C, H, W, device, images=None, image_dtype=torch.float32):
        self.host = {"questions": _pinned(B * S, torch.int32), "questionLengths": _pinned(B, torch.int32),
                     "answers": _pinned(B, torch.int32),
                     "images": _pinned((B if images is None else images) * C * H * W, image_dtype)}
        if images is not None:      # question b asks about image imageIndex[b] of the batch's k <= U
            self.host["imageIndex"] = _pinned(B, torch.int32)
        self.dev = {k: torch.empty(v.numel(), dtype=v.dtype, device=device) for k, v in self.host.items()}
        self.out = {"loss": _pinned(1, torch.float32), "gradNorm": _pinned(1, torch.float32),
                    "correctNum": _pinned(1, torch.int64), "predictions": _pinned(B, torch.int32)}
        self.copied = torch.cuda.Event()        # the H2D copies, on the copy stream
        self.done = torch.cuda.Event()          # the step and its D2H copies, on the step's stream
        self.busy = False


class TrainPipeline(object):
    """Training of the whole model from host buffers: what a caller with numpy or pinned-host batches uses in place of
    `MACnet.runBatch(train=True)`, with the same steps and the same results.

        pipe = TrainPipeline(model, shape=(B, S_max, H, W), depth=2)
        t = pipe.submit({"questions": int32 [B, S <= S_max] (0-padded), "questionLengths": int32 [B],
                         "answers": int32 [B], "images": fp32 [B, C, H, W]})
        res = pipe.result(t)      # {"loss", "correctNum", "acc", "gradNorm", "predictions" (pinned int32 [B])}

    Per batch, `submit` trims the questions to the longest one (as `runBatch` does, so the trainer's cells are keyed alike),
    stages the batch into the next of `depth` pinned buffers on `stage_threads` host threads (a pinned `images` tensor is
    copied from where it lies), copies it to the slot's device buffers on a copy stream, and enqueues
    `DPTrainer.train_step_full` on the caller's current stream behind that copy's event, with the NCHW features going
    straight into `Stem.forward_nchw`: the training ingest writes the fp32 NHWC tensor and layer 0's dropped-out patch
    matrix in one pass (`mac_ingest_nchw_train`).  The loss (mean over the batch), correct count, gradient norm and int32
    predictions go to pinned memory asynchronously; `result(ticket)` waits for that ticket's step only, and its values stay
    readable until `depth` further submits.  A slot's pinned and device buffers are written again only after the event of
    the step that read them.

    `submit` adds no synchronise of its own.  One remains inside the step: the cell reads the scalar logit biases with
    `.item()` (`MACParams.scalar`) after each optimizer step, so enqueueing step t waits for step t-1 to finish.  The
    staging and the copy of batch t run before that point, under step t-1's kernels.

    Batches in flight read and write the parameters: call `drain()` before evaluating (`runBatch(train=False)`,
    `ModelPipeline`, an EMA swap) or saving a checkpoint; training then continues with the next `submit` exactly as if it
    had not stopped.  With data-parallel training every rank runs its own pipeline over its shard (`global_batch = B * world`).
    A pinned `images` tensor must not be written until its ticket's result is read.

    Several questions per image: with `images=U` (1 <= U <= B) a batch carries k <= U distinct images and each question's
    image number, as `ModelPipeline(images=U)` takes them,

        pipe = TrainPipeline(model, shape=(B, S_max, H, W), depth=2, images=16)
        t = pipe.submit({"questions": ..., "questionLengths": ..., "answers": ..., "images": fp32 [k, C, H, W],
                         "imageIndex": int32 [B]})

    with 1 <= k <= U and every imageIndex[b] in [0, k).  The slots' pinned and device image buffers hold U images; only the k
    images are staged and copied, and the stem runs forward and backward over those k
    (`DPTrainer.full_forward_backward` with `imageIndex`: `mac_kb_gather`, `mac_kb_gather_bwd`).  The stem's input dropout is
    then drawn once per image, not once per question; everything after the stem is the step without an index.  With each
    rank's shard, each rank passes its own images and index.  Bad batches raise `ValueError` before anything is staged.

    Features stored in fp16: with `image_dtype=torch.float16` the batch's images must be fp16 host arrays (anything else
    raises `ValueError` before anything is staged); the pinned staging and device image buffers are fp16, half the bytes are
    staged and copied, and the step's ingest is `mac_ingest_nchw_train_f16`, which widens on the device: the step is bit for
    bit the default pipeline's step on the fp32 widening of the same features.  The default, `torch.float32`, widens an fp16
    batch on the host."""

    def __init__(self, model, shape, depth=2, stage_threads=None, images=None, image_dtype=torch.float32):
        B, S, H, W = [int(v) for v in shape]
        _check_image_dtype(image_dtype)
        t = model.trainer
        if t.stem is None:
            raise ValueError("the model's trainer has no stem: TrainPipeline trains the whole model")
        p = t.params
        C = model._stem.in_dim
        nfc = len([k for k in p.t if k.startswith("classifier/linearLayerfc_") and k.endswith("weights/weight")])
        self.A = int(p.t["classifier/linearLayerfc_%d/weights/weight" % (nfc - 1)].shape[1])
        if min(B, S, H, W) <= 0 or int(depth) < 1:
            raise ValueError("shape (B, S_max, H, W) and depth must be positive, got %r, depth = %r" % (shape, depth))
        if C % 64:
            raise ValueError("the image features have %d channels: mac_ingest_nchw_train needs a multiple of 64" % C)
        if images is not None and not (isinstance(images, int) and not isinstance(images, bool) and 1 <= images <= B):
            raise ValueError("images must be None or an int in 1..B = %d, got %r" % (B, images))
        self.images, self.image_dtype = images, image_dtype
        self.model, self.trainer, self.shape, self.C = model, t, (B, S, H, W), C
        self.stage_threads = int(stage_threads) if stage_threads else max(1, min(8, usable_cpus() // 2))
        self._pool = None
        if self.stage_threads > 1:
            from concurrent.futures import ThreadPoolExecutor
            self._pool = ThreadPoolExecutor(self.stage_threads)
        self.copy_stream = torch.cuda.Stream()
        self.slots = [_TrainSlot(B, S, C, H, W, p.flat.device, images, image_dtype) for _ in range(int(depth))]
        self._next = 0

    def _host(self, batch):
        """The batch's host tensors (with images=U also its image index, else None) and its longest question, checked against
        the pipeline's shape; ValueError before anything is enqueued."""
        B, S, H, W = self.shape
        if self.images is None and "imageIndex" in batch:
            raise ValueError("imageIndex is for a pipeline built with images=U")
        out = {}
        keys = (("questions", torch.int32), ("questionLengths", torch.int32), ("answers", torch.int32),
                ("images", torch.float32))
        if self.images is not None:
            keys += (("imageIndex", torch.int32),)
        for key, dtype in keys:
            if key not in batch:
                raise ValueError("the batch has no %s" % key)
            v = torch.as_tensor(batch[key])
            if v.device.type != "cpu":
                raise ValueError("%s must be host memory, got a tensor on %s" % (key, v.device))
            if key != "images" and (v.dtype.is_floating_point or v.dtype == torch.bool):
                raise ValueError("%s must hold integers, got %s" % (key, v.dtype))
            if key == "images" and self.image_dtype == torch.float16:
                _check_f16(v, "the batch's images")
                dtype = torch.float16
            out[key] = v if v.dtype == dtype and v.is_contiguous() else v.to(dtype).contiguous()
        q, ql, a, img = out["questions"], out["questionLengths"], out["answers"], out["images"]
        if q.dim() != 2 or q.shape[0] != B or not 1 <= q.shape[1] <= S:
            raise ValueError("questions must be [%d, S <= %d], got %s" % (B, S, tuple(q.shape)))
        for key, v in (("questionLengths", ql), ("answers", a)):
            if tuple(v.shape) != (B,):
                raise ValueError("%s must be [%d], got %s" % (key, B, tuple(v.shape)))
        idx = None
        if self.images is None:
            if tuple(img.shape) != (B, self.C, H, W):
                raise ValueError("images must be [%d, %d, %d, %d] (NCHW), got %s" % (B, self.C, H, W, tuple(img.shape)))
        else:
            if img.dim() != 4 or tuple(img.shape[1:]) != (self.C, H, W) or not 1 <= img.shape[0] <= self.images:
                raise ValueError("images must be [k, %d, %d, %d] (NCHW) with 1 <= k <= %d, got %s"
                                 % (self.C, H, W, self.images, tuple(img.shape)))
            idx = out["imageIndex"]
            if tuple(idx.shape) != (B,):
                raise ValueError("imageIndex must be [%d], got %s" % (B, tuple(idx.shape)))
            if int(idx.min()) < 0 or int(idx.max()) >= img.shape[0]:
                raise ValueError("imageIndex must lie in [0, %d) (the batch's images), got %d..%d"
                                 % (img.shape[0], int(idx.min()), int(idx.max())))
        longest = int(ql.max())
        if int(ql.min()) < 0 or not 1 <= longest <= q.shape[1]:
            raise ValueError("questionLengths must lie in [0, %d] with at least one question, got %d..%d"
                             % (q.shape[1], int(ql.min()), longest))
        if int(a.min()) < 0 or int(a.max()) >= self.A:
            raise ValueError("answers must lie in [0, %d), got %d..%d" % (self.A, int(a.min()), int(a.max())))
        return q, ql, a, img, idx, longest

    def _stage_images(self, dst, src):
        """Copy the flat `src` into the pinned `dst` of its dtype on the staging threads (numpy copies release the GIL)."""
        d, s = dst.numpy(), src.reshape(-1).numpy()
        if self._pool is None:
            np.copyto(d, s)
            return
        n, k = s.size, self.stage_threads
        cuts = [n * i // k for i in range(k + 1)]
        list(self._pool.map(lambda i: np.copyto(d[cuts[i]:cuts[i + 1]], s[cuts[i]:cuts[i + 1]]), range(k)))

    def submit(self, batch):
        """Stage, copy and enqueue one training step; returns its ticket."""
        q, ql, a, img, idx, S = self._host(batch)
        B = self.shape[0]
        n = img.numel()                         # B images, or the batch's k <= U with images=U
        tk = self._next
        slot = self.slots[tk % len(self.slots)]
        if slot.busy:
            slot.done.synchronize()             # the step that read this slot's buffers (depth submits back) has finished
        self._next = tk + 1
        h, dv = slot.host, slot.dev
        h["questions"][:B * S].view(B, S).copy_(q[:, :S])
        h["questionLengths"].copy_(ql)
        h["answers"].copy_(a)
        small = ("questionLengths", "answers")
        if idx is not None:
            h["imageIndex"].copy_(idx)
            small += ("imageIndex",)
        src = img.reshape(-1)
        if not img.is_pinned():
            self._stage_images(h["images"][:n], img)
            src = h["images"][:n]
        with torch.cuda.stream(self.copy_stream):
            dv["questions"][:B * S].copy_(h["questions"][:B * S], non_blocking=True)
            for k in small:
                dv[k].copy_(h[k], non_blocking=True)
            dv["images"][:n].copy_(src, non_blocking=True)
            slot.copied.record(self.copy_stream)
        stream = torch.cuda.current_stream()
        stream.wait_event(slot.copied)
        t = self.trainer
        data = {"questions": dv["questions"][:B * S].view(B, S), "questionLengths": dv["questionLengths"],
                "answers": dv["answers"], "images_nchw": dv["images"][:n].view(img.shape[0], self.C, *self.shape[2:])}
        if idx is not None:
            data["imageIndex"] = dv["imageIndex"]
        logits, losses = t.train_step_full((B, S), data, global_batch=B * t.world)
        self.model.macCell = t._cells[(B, S)][0]
        preds = torch.argmax(logits, dim=-1).to(torch.int32)                    # as runBatch computes them
        o = slot.out
        o["predictions"].copy_(preds, non_blocking=True)
        o["correctNum"].copy_((preds == data["answers"]).sum().view(1), non_blocking=True)
        o["loss"].copy_(losses.mean().view(1), non_blocking=True)
        o["gradNorm"].copy_(t.norm[:1], non_blocking=True)
        slot.done.record(stream)
        slot.busy = True
        return tk

    def result(self, ticket):
        """Block until the step of `ticket` is done: {"loss", "correctNum", "acc", "gradNorm"} as runBatch(train=True)
        reports them and "predictions", the pinned int32 [B] answer ids, valid until `depth` further submits."""
        if not self._next - len(self.slots) <= ticket < self._next:
            raise ValueError("ticket %r is not one of the last %d submits" % (ticket, len(self.slots)))
        slot = self.slots[ticket % len(self.slots)]
        slot.done.synchronize()
        o = slot.out
        n = int(o["correctNum"][0])
        return {"loss": float(o["loss"][0]), "correctNum": n, "acc": n / float(self.shape[0]),
                "gradNorm": float(o["gradNorm"][0]), "predictions": o["predictions"]}

    def predictions(self, out):
        """The predictions of a `result` as the model's `answer_decoder` spells them (ids without one)."""
        dec = self.model.decode
        return [dec(int(i)) if dec else int(i) for i in out["predictions"]]

    def drain(self):
        """Wait for every step in flight: afterwards the parameters, optimizer state and EMA are the last step's."""
        for s in self.slots:
            if s.busy:
                s.done.synchronize()
