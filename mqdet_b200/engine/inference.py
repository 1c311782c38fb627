"""Inference engine: the forward captured ONCE as a CUDA graph and replayed per batch, inputs prefetched on a copy stream.

It is the counterpart of the reference's evaluation loop (maskrcnn_benchmark/engine/inference.py:435-470,
``for batch in data_loader: output = model(images.to(device), captions=..., positive_map=...)``): same inputs (a batch of
images + one prompt), same outputs (``list[BoxList]`` per batch), but

  * the ~600 kernel launches of a forward are recorded into one ``cudaGraph`` (fixed shapes: batch size, padded image
    size and prompt do not change inside an evaluation run), so a step costs one graph launch on the host instead of
    ~600 ctypes calls — the per-rank host jitter no longer reaches the GPU timeline, and the small text-stream kernels
    are never starved by the launch rate;
  * the host->device copy of batch s+1 (pinned memory -> a second device buffer, on a copy stream) overlaps the replay of
    batch s; the packed fixed-shape result ``[B, max_out + 1, 6]`` (detections + count row) is the ONE device->host copy;
  * with ``torch.distributed`` initialised, the ONE collective of the data path (all-gather of the packed results over
    NCCL / NVLink) and the device->host copies run on a separate RESULT stream behind the forward: the next replay starts
    without waiting for the slowest rank to reach the collective.  The reference gathers the predictions of all ranks ONCE
    per evaluation (engine/inference.py:294 -> utils/comm.py:61-102, a pickled variable-length all_gather); here the packed
    fixed-shape results of ``gather_every`` consecutive steps accumulate in a device ring and are exchanged by one
    ``all_gather_into_tensor`` (plus a final ``flush()``): an NCCL kernel that sits on an SM waiting for a peer takes that SM
    away from the persistent one-CTA-per-SM kernels of the next forward, so the collective is kept rare, not per step.

Nothing here computes: it is stream / graph / buffer plumbing around ``GeneralizedVLRCNN_New.forward_device``.

``run_batches`` / ``run_images`` of both engines take the reference's test-loader batches instead: padded batches of differently
sized images, whose batch size and padded shape change from batch to batch (``engine/batches.py::reference_test_batches``).  They
keep one CUDA graph per padded batch shape (B, Hp, Wp) in ``ShapeGraphs``; the image sizes are not part of a graph, they travel in a
device table the forward reads.  ``ChunkedEngine`` does the same for the chunked many-category forward (LVIS) of either detector.
"""
import random
import time
from collections import OrderedDict

import torch
import torch.distributed as dist

from .. import parallel
from .._lib import MqdetError
from ..structures.bounding_box import boxlists_from_packed
from ..structures.image_list import ImageList


class _ShapeGraphEngine:
    """What the three engines share: the checks of the model, and ``run_batches`` / ``run_images`` / ``close`` over the
    ``ShapeGraphs`` of the engine's forward, built on first use.  The forward is the single-prompt ``forward_device`` of either
    detector; ``ChunkedEngine`` replaces it with its chunked forward."""
    n_chunks = 1

    def __init__(self, model, *, use_graph, warmup, max_graphs):
        # vision-only evaluation: at TEXT_DROPOUT >= 1 the masked ids are part of the captured prompt state
        self.mask_rate = model.text_mask_rate()
        if 0 < self.mask_rate < 1:
            raise NotImplementedError("VISION_QUERY.TEXT_DROPOUT < 1 with VISION_QUERY.MASK_DURING_INFERENCE: every forward draws new "
                                      "token masks, which a replayed graph cannot do; use the eager forward")
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise MqdetError(f"{type(self).__name__}: the model must live on a CUDA device (no CPU fallback)")
        self.model = model
        self.use_graph, self.warmup, self.max_graphs = bool(use_graph), max(1, int(warmup)), max_graphs
        self.batches = None                     # ShapeGraphs of run_batches / run_images, built on first use

    def _refuse(self, what):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            raise NotImplementedError(f"{what} runs on one GPU: under GroupedBatchSampler the ranks' batch counts and tail sizes "
                                      "differ, so the ranks would not reach the same steps; run it per rank without a process group, "
                                      "or use run() with one batch shape")

    def _graph_forward(self, il, wh):
        return self.model.forward_device(il, self.captions, self.positive_map, img_wh=wh)["det_packed"]

    def _after_replay(self, state):
        """The draws of the eager forward at TEXT_DROPOUT >= 1, so that Python's random advances as in the reference (MQ-GLIP only:
        MQ-GroundingDINO's rate is 0)."""
        self.model.draw_text_masks(state[0]["has"], self.mask_rate)

    def _shape_graphs(self):
        if self.batches is None:
            self.batches = ShapeGraphs(self.model, self._graph_forward, self.n_chunks, use_graph=self.use_graph, warmup=self.warmup,
                                       max_graphs=self.max_graphs, after_replay=self._after_replay if self.mask_rate > 0 else None)
        return self.batches

    def run_batches(self, batches):
        """batches: iterable of ``ImageList`` (a pinned-host or device fp32 tensor [B, 3, Hp, Wp] + ``image_sizes``), e.g. the
        reference's test-loader batches -> yields list[BoxList] per batch, each at its image's own size, equal bit for bit to the
        eager forward (``model(il, ...)`` / ``model.forward_chunked(il, ...)``).  One graph per (B, Hp, Wp), captured the first time
        that shape comes (see ``ShapeGraphs``); the upload of batch s+1 overlaps the forward of batch s."""
        self._refuse("run_batches")
        return self._shape_graphs().run_batches(batches)

    def run_images(self, images_u8, index_batches):
        """Decoded uint8 HWC RGB images + the index lists of ``reference_test_batches`` -> yields list[BoxList] per index list in
        original-image coordinates, equal to the test transform followed by the eager forward.  The upload and the test transform run
        on the copy stream, straight into the staging buffer the next forward reads."""
        self._refuse("run_images")
        return self._shape_graphs().run_images(images_u8, index_batches)

    def close(self):
        """Drop the graphs of ``run_batches`` / ``run_images``."""
        if self.batches is not None:
            self.batches.close()
            self.batches = None


class InferenceEngine(_ShapeGraphEngine):
    def __init__(self, model, captions, positive_map, batch_shape=None, image_sizes=None, *, use_graph=True, gather=True, warmup=2,
                 gather_every=8, max_graphs=None):
        """model: GeneralizedVLRCNN_New (eval, on its CUDA device); captions / positive_map: the prompt of the run;
        batch_shape: (B, 3, H, W) of the padded batch tensor; image_sizes: [(h, w)] * B un-padded sizes;
        gather_every: steps whose packed results are exchanged by one all-gather (N > 1).
        Without ``batch_shape`` / ``image_sizes`` nothing is captured up front and only ``run_batches`` / ``run_images`` serve;
        ``max_graphs`` bounds their live graphs (default ``ShapeGraphs.MAX_GRAPHS``)."""
        super().__init__(model, use_graph=use_graph, warmup=warmup, max_graphs=max_graphs)
        self.captions, self.positive_map = captions, positive_map
        self.graphs, self.outs = [None, None], [None, None]
        self.max_out = model.max_out()
        if batch_shape is None or image_sizes is None:
            if batch_shape is not None or image_sizes is not None:
                raise ValueError("InferenceEngine: batch_shape and image_sizes go together")
            return
        self.image_sizes = [tuple(s) for s in image_sizes]
        self.B = int(batch_shape[0])
        self.world = dist.get_world_size() if (gather and dist.is_available() and dist.is_initialized()) else 1
        self.stage = [torch.empty(tuple(batch_shape), dtype=torch.float32, device=self.dev) for _ in range(2)]
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.up_done = [torch.cuda.Event(), torch.cuda.Event()]   # upload into stage[k] finished
        self.fw_done = [torch.cuda.Event(), torch.cuda.Event()]   # the forward that read stage[k] finished
        # local packed result of a step -> pinned host (the BoxLists of `run`)
        self.host = [torch.empty((self.B, self.max_out + 1, 6), dtype=torch.float32).pin_memory() for _ in range(2)]
        self.d2h_done = [torch.cuda.Event(), torch.cuda.Event()]
        # result stream: ring append (+ all-gather every G steps, N > 1) + device->host copies of step s while the main stream
        # already runs step s+1
        self.result_stream = torch.cuda.Stream(device=self.dev)
        self.res_done = [torch.cuda.Event(), torch.cuda.Event()]  # everything that read outs[k]["packed"] finished
        self.G = max(1, int(gather_every))
        self.ring_fill = 0            # steps appended since the last exchange
        self.exchanges = 0            # all-gathers issued
        self.gather_done = torch.cuda.Event()
        if self.world > 1:
            self.ring = torch.zeros((self.G, self.B, self.max_out + 1, 6), dtype=torch.float32, device=self.dev)
            self.gathered = torch.zeros((self.world, self.G, self.B, self.max_out + 1, 6), dtype=torch.float32, device=self.dev)
            self.gathered_host = torch.zeros(tuple(self.gathered.shape), dtype=torch.float32).pin_memory()
        else:
            self.ring = self.gathered = self.gathered_host = None
        main = torch.cuda.current_stream(self.dev)
        for ev in self.fw_done + self.res_done + [self.gather_done]:
            ev.record(main)
        # warm-up on the real buffers: fills every per-prompt / per-shape cache (token ids, selected queries, index tables,
        # level tables, fp16 weight copies, tensor maps, shared-memory opt-ins) so that the capture sees launches only
        for _ in range(max(1, warmup)):
            for k in range(2):
                self.outs[k] = self._forward(k)
                self._collect(k, to_host=False)
        self.flush()
        torch.cuda.synchronize(self.dev)
        if self.use_graph:
            pool = None
            for k in range(2):  # one graph per staging buffer (the input address is baked into the graph); the two graphs
                g = torch.cuda.CUDAGraph()  # are only ever replayed one after the other, so they share a memory pool
                with torch.cuda.graph(g, pool=pool):
                    self.outs[k] = self._forward(k)
                pool = g.pool()
                self.graphs[k] = g
            torch.cuda.synchronize(self.dev)

    def _forward(self, k):
        out = self.model.forward_device(ImageList(self.stage[k], self.image_sizes), self.captions, self.positive_map)
        return {"packed": out["det_packed"], "raw": out}

    def _collect(self, k, to_host=True):
        """On the result stream, behind the forward of slot k: append the packed result to the exchange ring (N > 1; the ONE
        collective of the data path runs when the ring is full), and the device->host copy of the local result."""
        main = torch.cuda.current_stream(self.dev)
        self.fw_done[k].record(main)
        rs = self.result_stream
        with torch.cuda.stream(rs):
            rs.wait_event(self.fw_done[k])
            res = self.outs[k]["packed"]
            if self.world > 1:
                self.ring[self.ring_fill].copy_(res, non_blocking=True)
                self.ring_fill += 1
                if self.ring_fill == self.G:
                    self._exchange(rs)
            if to_host:
                self.host[k].copy_(res, non_blocking=True)
                self.d2h_done[k].record(rs)
            self.res_done[k].record(rs)
        return res

    def _exchange(self, rs):
        """(result stream) all-gather of the ring -> gathered [world, G, B, max_out + 1, 6] -> pinned host copy."""
        parallel.all_gather_packed(self.ring.view(self.G * self.B, self.max_out + 1, 6),
                                   out=self.gathered.view(self.world * self.G * self.B, self.max_out + 1, 6))
        self.gathered_host.copy_(self.gathered, non_blocking=True)
        self.gather_done.record(rs)
        self.last_exchange_steps = self.ring_fill
        self.ring_fill = 0
        self.exchanges += 1

    def flush(self):
        """Exchange a partly filled ring (end of an evaluation run; every rank must call it the same number of times)."""
        if self.world > 1 and self.ring_fill > 0:
            with torch.cuda.stream(self.result_stream):
                self._exchange(self.result_stream)

    def gathered_results(self):
        """Pinned host tensor [world, steps, B, max_out + 1, 6] of the LAST exchange (waits for its copy), rank-major."""
        if self.world == 1:
            return None
        self.gather_done.synchronize()
        return self.gathered_host[:, :self.last_exchange_steps]

    # -- one step on staging buffer k: (graph replay | eager forward) -> [all-gather ->] async D2H of the packed result ----
    def _step(self, k, to_host):
        main = torch.cuda.current_stream(self.dev)
        main.wait_event(self.up_done[k])
        main.wait_event(self.res_done[k])   # the previous result of this slot has been gathered / copied out
        if self.use_graph:
            self.graphs[k].replay()
            if self.mask_rate > 0:   # the draws of the eager forward, so that Python's random advances as in the reference
                self.model.draw_text_masks(self.model._prompt["has"], self.mask_rate)
        else:
            self.outs[k] = self._forward(k)
        self._collect(k, to_host)
        return self.outs[k]

    def _launch(self, k):
        return self._step(k, True)

    def _upload(self, k, images_host):
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(self.fw_done[k])     # stage[k] is no longer being read
            self.stage[k].copy_(images_host, non_blocking=True)
            self.up_done[k].record(self.copy_stream)

    def device_step(self, images_dev=None, k=0):
        """Device-resident step (bench `value`): optional device->device refresh of the input, then one replay; on the result
        stream the packed result joins the exchange ring (N > 1).  No host traffic, no synchronisation."""
        if images_dev is not None and images_dev.data_ptr() != self.stage[k].data_ptr():
            self.stage[k].copy_(images_dev, non_blocking=True)
        self.up_done[k].record(torch.cuda.current_stream(self.dev))
        o = self._step(k, False)
        return {"packed": o["packed"], "raw": o["raw"]}

    def close(self):
        """Drain both streams and drop the captured graphs (call before destroying the process group)."""
        torch.cuda.synchronize(self.dev)
        for g in self.graphs:
            if g is not None:
                g.reset()
        self.graphs = [None, None]
        self.outs = [None, None]
        self.use_graph = False
        super().close()
        torch.cuda.synchronize(self.dev)

    def run(self, batches):
        """batches: iterable of pinned (or pageable) HOST tensors [B, 3, H, W] -> yields list[BoxList] per batch, in order.
        Two batches are in flight: the upload of batch s+1 overlaps the forward of batch s, and the forward of batch s+1 is
        already queued when the host turns the packed result of batch s into BoxLists."""
        it = iter(batches)
        try:
            cur = next(it)
        except StopIteration:
            return
        k = 0
        self._upload(k, cur)
        self._launch(k)
        while True:
            try:
                nxt = next(it)
            except StopIteration:
                nxt = None
            if nxt is not None:
                self._upload(k ^ 1, nxt)
                self._launch(k ^ 1)
            if nxt is None:
                self.flush()  # the tail of the run reaches the other ranks
            self.d2h_done[k].synchronize()   # the LOCAL images' packed result is in pinned host buffer k
            yield boxlists_from_packed(self.host[k], self.image_sizes)
            if nxt is None:
                return
            k ^= 1


class GroundingDINOEngine(_ShapeGraphEngine):
    """The same idea for ``mqdet_b200.modeling.groundingdino.groundingdino.GroundingDINO`` (BASELINE config 4): the whole forward
    (≈ 780 kernels at 2 images) recorded once as a CUDA graph over a static input buffer and replayed per batch; pinned host images in,
    ``list[BoxList]`` out, and — with ``torch.distributed`` initialised — ONE all-gather of the packed ``[B, num_queries + 1, 6]`` result
    per step (``parallel.all_gather_packed``), issued after the replay, outside the graph.

        eng = GroundingDINOEngine(model, captions, positive_map, batch_shape=(2, 3, 800, 1344), image_sizes=[(800, 1333)] * 2)
        for boxlists in eng.run(host_batches): ...
    """

    def __init__(self, model, captions, positive_map, batch_shape=None, image_sizes=None, *, use_graph=True, gather=True, warmup=2,
                 max_graphs=None):
        """Without ``batch_shape`` / ``image_sizes`` nothing is captured up front and only ``run_batches`` / ``run_images`` serve
        (one graph per padded shape, at most ``max_graphs`` live, default ``ShapeGraphs.MAX_GRAPHS``)."""
        super().__init__(model, use_graph=use_graph, warmup=warmup, max_graphs=max_graphs)
        self.captions, self.positive_map = captions, positive_map
        self.graph, self.static_out, self.note = None, None, "eager launches"
        if batch_shape is None or image_sizes is None:
            if batch_shape is not None or image_sizes is not None:
                raise ValueError("GroundingDINOEngine: batch_shape and image_sizes go together")
            return
        self.image_sizes = [tuple(s) for s in image_sizes]
        self.B, self.nq = int(batch_shape[0]), int(model.num_queries)
        self.world = dist.get_world_size() if (gather and dist.is_available() and dist.is_initialized()) else 1
        self.static_in = torch.zeros(tuple(batch_shape), dtype=torch.float32, device=self.dev)
        self.images = ImageList(self.static_in, self.image_sizes)
        self.host = torch.empty((self.B, self.nq + 1, 6), dtype=torch.float32).pin_memory()
        self.gathered = torch.empty((self.world * self.B, self.nq + 1, 6), dtype=torch.float32, device=self.dev) if self.world > 1 else None
        self.graph, self.static_out, self.note = None, None, "eager launches"
        for _ in range(max(1, warmup)):          # fills the per-prompt / per-geometry caches, fp16 weight copies, tensor maps
            model.forward_device(self.images, captions, positive_map)
        torch.cuda.synchronize(self.dev)
        if use_graph:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self.static_out = model.forward_device(self.images, captions, positive_map)["det_packed"]
                self.graph, self.note = g, "cuda-graph replay of the whole forward"
            except Exception as e:  # noqa: BLE001 - capture is an optimisation; the eager path is the same arithmetic
                self.graph, self.note = None, f"eager launches (graph capture failed: {type(e).__name__}: {str(e)[:120]})"
                torch.cuda.synchronize(self.dev)

    @torch.no_grad()
    def step_device(self, x=None):
        """One forward over ``x`` (a device or pinned-host batch; None = whatever the input buffer holds) -> the device-resident
        packed result of THIS rank ([B, nq + 1, 6]) or, N > 1, of all ranks ([world * B, nq + 1, 6], rank-major)."""
        if x is not None:
            self.static_in.copy_(x, non_blocking=True)
        if self.graph is not None:
            self.graph.replay()
            det = self.static_out
        else:
            det = self.model.forward_device(self.images, self.captions, self.positive_map)["det_packed"]
        if self.world > 1:
            return parallel.all_gather_packed(det.contiguous(), out=self.gathered)
        return det

    @torch.no_grad()
    def run(self, host_batches):
        """host_batches: iterable of pinned fp32 [B,3,H,W] tensors -> yields ``list[BoxList]`` of the LOCAL images per batch."""
        rank = dist.get_rank() if self.world > 1 else 0
        for hb in host_batches:
            det = self.step_device(hb)
            local = det[rank * self.B:(rank + 1) * self.B] if self.world > 1 else det
            self.host.copy_(local, non_blocking=True)
            torch.cuda.current_stream(self.dev).synchronize()
            yield boxlists_from_packed(self.host, self.image_sizes)


class ChunkedEngine(_ShapeGraphEngine):
    """Chunked evaluation of a many-category vocabulary (LVIS: TEST.CHUNKED_EVALUATION 40 turns 1203 classes into 31 prompts) through
    CUDA graphs, for either detector (``GeneralizedVLRCNN_New`` or ``GroundingDINO``; dispatched on its ``forward_chunked_device``).
    The reference evaluates LVIS at TEST.IMS_PER_BATCH 1, every image its own batch at its own padded size; here one graph per
    padded batch shape holds every pass of every chunk, so an image costs one replay instead of ~780 launches per pass.

        eng = ChunkedEngine(model, chunk_captions, chunk_positive_maps, chunks_per_pass=8)
        for boxlists in eng.run_batches(image_lists): ...             # padded ImageLists, e.g. one image each
        for boxlists in eng.run_images(images_u8, index_batches): ... # decoded uint8 + reference_test_batches index lists
        eng.stats(); eng.close()

    Each BoxList holds an image's per-chunk detections concatenated in chunk order with their global labels: what
    ``forward_chunked`` returns and the reference's ``concate_box_list`` makes (engine/inference.py:704-706), bit for bit."""

    # Live graphs by default.  A COCO-like set at 800 / 1333 has 43 padded shapes: one side at 800 and the other in 32-pixel steps
    # up to 1344, both orientations (35), plus the shapes whose long side is capped at 1333 (8).  Measured over all 43 at 31 chunks
    # of 40 classes, 8 per pass, one image per batch (tools/prof_chunked_engine.py --all-shapes, H100 80GB HBM3, 700 W; DESIGN.md
    # section 5): 43 captures, no eviction; per graph 8.3 MB allocated and 16-19 MB reserved beyond the staging buffers (the first
    # few graphs of a run reserve ~110 MB each, later ones reuse the shared pool); peak max_memory_allocated 6.7 GB for
    # MQ-GroundingDINO-T, 4.0 GB for MQ-GLIP-T.  48 leaves room for a few more shapes at well under 1 GB.
    MAX_GRAPHS = 48

    def __init__(self, model, chunk_captions, chunk_positive_maps, chunks_per_pass=8, max_graphs=None, *, use_graph=True, warmup=2):
        if not hasattr(model, "forward_chunked_device"):
            raise TypeError(f"ChunkedEngine: {type(model).__name__} has no forward_chunked_device")
        if len(chunk_captions) != len(chunk_positive_maps) or not chunk_captions:
            raise ValueError("ChunkedEngine: one positive map per chunk caption, at least one chunk")
        if int(chunks_per_pass) < 1:
            raise ValueError(f"chunks_per_pass must be >= 1, got {chunks_per_pass}")
        self.model = model
        self._refuse("ChunkedEngine")
        super().__init__(model, use_graph=use_graph, warmup=warmup, max_graphs=self.MAX_GRAPHS if max_graphs is None else max_graphs)
        self.captions, self.positive_maps = list(chunk_captions), list(chunk_positive_maps)
        self.chunks_per_pass, self.n_chunks = int(chunks_per_pass), len(self.captions)

    def _refuse(self, what):
        super()._refuse(what)
        # a capture must find every chunk group cached: rebuilding one reads a count on the host and uploads small tables
        if not self.model.cache_chunk_groups:
            raise NotImplementedError("ChunkedEngine needs model.cache_chunk_groups = True: a graph can only replay chunk-group "
                                      "state built before its capture")

    def _graph_forward(self, il, wh):
        pk = self.model.forward_chunked_device(il, self.captions, self.positive_maps, self.chunks_per_pass, img_wh=wh)["det_packed"]
        return pk.transpose(0, 1).reshape(pk.shape[1], -1, 6)      # [B, n_chunks * rows, 6]

    def _after_replay(self, state):
        read = state[-1]
        self.model.draw_chunk_text_masks(read["states"], read["B"], self.mask_rate)

    def stats(self):
        """Captures, seconds spent in warm-ups and captures, distinct shapes seen, evictions, graphs live."""
        return self._shape_graphs().stats()


class _Graph:
    __slots__ = ("graph", "state")

    def __init__(self, graph, state):
        self.graph, self.state = graph, state


class ShapeGraphs:
    """CUDA graphs of one detector forward keyed by the padded batch shape (B, Hp, Wp), for padded batches of differently sized
    images.

    Buffers, all allocated outside the graphs' memory pool, each sized for the largest batch the config allows (TEST.IMS_PER_BATCH
    images of MAX_SIZE_TEST rounded up to SIZE_DIVISIBILITY on both sides; a larger batch is refused):
      * two staging slots, each an input buffer, a device (w, h) size table and a pinned host result buffer.  The copy stream
        writes a batch's images and sizes into slot s % 2 while the forward of the batch before runs;
      * the graphs' own input, size table and result buffer.  Before a replay the main stream copies the slot into them (a
        device-to-device copy of the batch, well under 1% of a forward); every graph reads the input and the table at the
        addresses it was captured with and ends by copying its packed result into the result buffer.  So one graph serves both
        slots, and a shape is captured once.
    Because every graph's result leaves the pool before the graph ends, the pool holds only scratch that a replay writes before
    it reads it: all graphs share it, and they may replay in the order of the data rather than the order of capture.

    A new shape gets ``warmup`` eager forwards (they fill the per-prompt / per-batch-size caches and the lazy kernel set-up), then
    a capture.  The single-entry caches of the model (prompt state, token map, GCP tables) are replaced when another batch size
    comes; each graph keeps the entries it captured (``model.graph_state()``) for as long as it lives, so a replay never reads a
    freed block.  Keeping them with the graph rather than keying the caches ties their lifetime to the one thing that reads them,
    with no second bound or eviction policy to keep in step.  At most ``max_graphs`` graphs live; the least recently used one
    is dropped first.  A short tail batch is its own shape: padding it with dummy images would change its results in the last
    bits, since batch elements agree only to rounding."""

    # Live graphs by default.  Measured per captured graph (tools/prof_mixed_batches.py, H100 80GB HBM3, 700 W; DESIGN.md section
    # 5): MQ-GLIP-T 16 MB allocated / 183 MB reserved, MQ-GroundingDINO-T 43 / 113 MB.  32 graphs hold at most ~6 GB, and cover
    # the padded shapes of a COCO-sized set at 800 / 1333 (one side at 800, the other in 32-pixel steps, per orientation).
    MAX_GRAPHS = 32

    def __init__(self, model, forward, n_chunks=1, *, use_graph=True, warmup=1, max_graphs=None, after_replay=None):
        """forward(ImageList, img_wh fp32 [B, 2] device) -> packed fp32 [B, n_chunks * (model.max_out() + 1), 6] device result
        (``boxlists_from_packed`` turns it into BoxLists); after_replay(graph state): host work an eager forward would also do."""
        cfg = model.cfg
        self.model, self.forward, self.n_chunks = model, forward, int(n_chunks)
        self.rows = self.n_chunks * (model.max_out() + 1)
        self.after_replay = after_replay
        self.use_graph, self.warmup = bool(use_graph), max(1, int(warmup))
        self.max_graphs = self.MAX_GRAPHS if max_graphs is None else int(max_graphs)
        if self.max_graphs < 1:
            raise ValueError(f"max_graphs must be >= 1, got {max_graphs}")
        self.dev = next(model.parameters()).device
        div = int(cfg.DATALOADER.SIZE_DIVISIBILITY)
        side = int(cfg.INPUT.MAX_SIZE_TEST)
        side = -(-side // div) * div if div > 0 else side
        self.max_B, self.max_hw = int(cfg.TEST.IMS_PER_BATCH), (side, side)
        n = self.max_B * 3 * side * side
        f32 = dict(dtype=torch.float32, device=self.dev)
        self.slot_in = [torch.empty((n,), **f32) for _ in range(2)]
        self.slot_wh = [torch.empty((self.max_B, 2), **f32) for _ in range(2)]
        self.host = [torch.empty((self.max_B, self.rows, 6), dtype=torch.float32).pin_memory() for _ in range(2)]
        self.g_in, self.g_wh = torch.empty((n,), **f32), torch.zeros((self.max_B, 2), **f32)
        self.g_res = torch.empty((self.max_B, self.rows, 6), **f32)
        self.buffer_bytes = 4 * (3 * n + 3 * 2 * self.max_B + self.max_B * self.rows * 6)
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.up_done = [torch.cuda.Event() for _ in range(2)]     # images + sizes of slot k uploaded
        self.fw_done = [torch.cuda.Event() for _ in range(2)]     # slot k copied into the graph input: it may be overwritten
        self.d2h_done = [torch.cuda.Event() for _ in range(2)]    # packed result of slot k in its pinned host buffer
        main = torch.cuda.current_stream(self.dev)
        for ev in self.fw_done + self.d2h_done:
            ev.record(main)
        self.pool = torch.cuda.graph_pool_handle()
        self.graphs = OrderedDict()
        self.captures, self.evictions, self.capture_s = 0, 0, 0.0
        self.keys = set()

    def close(self):
        torch.cuda.synchronize(self.dev)
        for e in self.graphs.values():
            e.graph.reset()
        self.graphs.clear()

    def stats(self):
        """Captures, seconds spent in warm-ups and captures, distinct shapes seen, evictions, graphs live."""
        return {"captures": self.captures, "capture_s": self.capture_s, "keys": len(self.keys), "evictions": self.evictions,
                "live": len(self.graphs)}

    # -- staging (copy stream) -------------------------------------------------------------------------------------------
    def _check_shape(self, B, Hp, Wp):
        if not (1 <= B <= self.max_B and Hp <= self.max_hw[0] and Wp <= self.max_hw[1]):
            raise MqdetError(f"batch [{B}, 3, {Hp}, {Wp}] exceeds the staging buffers [{self.max_B}, 3, {self.max_hw[0]}, "
                             f"{self.max_hw[1]}] (TEST.IMS_PER_BATCH images of INPUT.MAX_SIZE_TEST rounded up to SIZE_DIVISIBILITY)")

    def _stage_sizes(self, k, image_sizes):
        """(copy stream) the (w, h) table of the batch -> slot k."""
        wh = torch.tensor([[float(w), float(h)] for h, w in image_sizes], dtype=torch.float32).pin_memory()
        self.slot_wh[k][:len(image_sizes)].copy_(wh, non_blocking=True)

    def _stage_batch(self, k, il):
        x = il.tensors
        if x.dim() != 4 or x.shape[1] != 3 or x.dtype != torch.float32:
            raise MqdetError(f"run_batches: fp32 [B, 3, Hp, Wp] images required (got {x.dtype} {tuple(x.shape)})")
        B, _, Hp, Wp = x.shape
        if len(il.image_sizes) != B:
            raise MqdetError(f"run_batches: {len(il.image_sizes)} image sizes for {B} images")
        self._check_shape(B, Hp, Wp)
        cs = self.copy_stream
        produced = torch.cuda.Event()
        produced.record(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(cs):
            cs.wait_event(self.fw_done[k])                       # the forward before has taken slot k's contents
            if x.is_cuda:
                cs.wait_event(produced)
                x.record_stream(cs)
            self.slot_in[k][:x.numel()].view(B, 3, Hp, Wp).copy_(x, non_blocking=True)
            self._stage_sizes(k, il.image_sizes)
            self.up_done[k].record(cs)
        return (B, Hp, Wp), [tuple(s) for s in il.image_sizes], None

    def _stage_images(self, k, tf, images_u8, idx):
        cs = self.copy_stream
        produced = torch.cuda.Event()                            # device images may come from work on the main stream
        produced.record(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(cs):
            cs.wait_event(self.fw_done[k])
            cs.wait_event(produced)
            il, orig = tf([images_u8[i] for i in idx], self.dev, mixed_sizes=True, out=self.slot_in[k])
            B, _, Hp, Wp = il.tensors.shape
            self._check_shape(B, Hp, Wp)
            self._stage_sizes(k, il.image_sizes)
            self.up_done[k].record(cs)
        return (B, Hp, Wp), il.image_sizes, orig

    # -- one forward (main stream) ---------------------------------------------------------------------------------------
    def _graph_input(self, key):
        B, Hp, Wp = key
        return self.g_in[:B * 3 * Hp * Wp].view(B, 3, Hp, Wp), self.g_wh[:B]

    def _capture(self, key, image_sizes):
        x, wh = self._graph_input(key)
        il = ImageList(x, image_sizes)
        t0 = time.perf_counter()
        for i in range(self.warmup):
            self.forward(il, wh)
            if i == 0:   # the first forward draws what an eager forward of this batch draws (vision-only masks, query picks);
                rstate = random.getstate()   # the further warm-ups and the capture must not advance Python's random
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, pool=self.pool):
            self.g_res[:key[0]].copy_(self.forward(il, wh))
        state = self.model.graph_state()
        random.setstate(rstate)
        e = self.graphs[key] = _Graph(g, state)
        while len(self.graphs) > self.max_graphs:   # evicted after the capture: the shared pool must stay in use meanwhile
            _, old = self.graphs.popitem(last=False)
            old.graph.reset()
            self.evictions += 1
        torch.cuda.synchronize(self.dev)
        self.capture_s += time.perf_counter() - t0
        self.captures += 1
        return e

    def _launch(self, k, key, image_sizes):
        main = torch.cuda.current_stream(self.dev)
        main.wait_event(self.up_done[k])
        main.wait_event(self.d2h_done[k])                       # slot k's host buffer has been read by the previous batch
        B, Hp, Wp = key
        n = B * 3 * Hp * Wp
        self.g_in[:n].copy_(self.slot_in[k][:n], non_blocking=True)
        self.g_wh[:B].copy_(self.slot_wh[k][:B], non_blocking=True)
        self.fw_done[k].record(main)
        self.keys.add(key)
        if self.use_graph:
            e = self.graphs.get(key)
            fresh = e is None
            if fresh:
                e = self._capture(key, image_sizes)
            else:
                self.graphs.move_to_end(key)
            e.graph.replay()
            if self.after_replay is not None and not fresh:   # a new shape's first warm-up forward did this batch's host work
                self.after_replay(e.state)
        else:
            x, wh = self._graph_input(key)
            self.g_res[:B].copy_(self.forward(ImageList(x, image_sizes), wh))
        self.host[k][:B].copy_(self.g_res[:B], non_blocking=True)
        self.d2h_done[k].record(main)

    def _results(self, k, B, image_sizes):
        self.d2h_done[k].synchronize()
        return boxlists_from_packed(self.host[k][:B], image_sizes, self.n_chunks)

    def _run(self, items, stage):
        """Two batches in flight: batch s+1 is staged and its forward queued before the host turns batch s into BoxLists."""
        it = iter(items)
        first = next(it, None)
        if first is None:
            return
        k = 0
        cur = stage(k, first)
        self._launch(k, cur[0], cur[1])
        while True:
            item = next(it, None)
            nxt = None
            if item is not None:
                nxt = stage(k ^ 1, item)
                self._launch(k ^ 1, nxt[0], nxt[1])
            key, sizes, orig = cur
            res = self._results(k, key[0], sizes)
            yield res if orig is None else [bl.resize(o) for bl, o in zip(res, orig)]
            if nxt is None:
                return
            k ^= 1
            cur = nxt

    @torch.no_grad()
    def run_batches(self, batches):
        yield from self._run(batches, self._stage_batch)

    @torch.no_grad()
    def run_images(self, images_u8, index_batches):
        from .transforms import TestTransform
        tf = TestTransform(self.model.cfg)
        yield from self._run(index_batches, lambda k, idx: self._stage_images(k, tf, images_u8, idx))
