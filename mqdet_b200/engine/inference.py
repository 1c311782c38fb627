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
"""
import torch
import torch.distributed as dist

from .. import parallel
from .._lib import MqdetError
from ..structures.image_list import ImageList


class InferenceEngine:
    def __init__(self, model, captions, positive_map, batch_shape, image_sizes, *, use_graph=True, gather=True, warmup=2,
                 gather_every=8):
        """model: GeneralizedVLRCNN_New (eval, on its CUDA device); captions / positive_map: the prompt of the run;
        batch_shape: (B, 3, H, W) of the padded batch tensor; image_sizes: [(h, w)] * B un-padded sizes;
        gather_every: steps whose packed results are exchanged by one all-gather (N > 1)."""
        # vision-only evaluation: at TEXT_DROPOUT >= 1 the masked ids are part of the captured prompt state
        self.mask_rate = model.text_mask_rate()
        if 0 < self.mask_rate < 1:
            raise NotImplementedError("VISION_QUERY.TEXT_DROPOUT < 1 with VISION_QUERY.MASK_DURING_INFERENCE: every forward draws new "
                                      "token masks, which a replayed graph cannot do; use forward_device")
        self.model = model
        self.captions, self.positive_map = captions, positive_map
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise MqdetError("InferenceEngine: the model must live on a CUDA device (no CPU fallback)")
        self.image_sizes = [tuple(s) for s in image_sizes]
        self.B = int(batch_shape[0])
        self.world = dist.get_world_size() if (gather and dist.is_available() and dist.is_initialized()) else 1
        self.stage = [torch.empty(tuple(batch_shape), dtype=torch.float32, device=self.dev) for _ in range(2)]
        self.copy_stream = torch.cuda.Stream(device=self.dev)
        self.up_done = [torch.cuda.Event(), torch.cuda.Event()]   # upload into stage[k] finished
        self.fw_done = [torch.cuda.Event(), torch.cuda.Event()]   # the forward that read stage[k] finished
        self.graphs = [None, None]
        self.outs = [None, None]
        self.max_out = model.max_out()
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
        self.use_graph = bool(use_graph)
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
        torch.cuda.synchronize(self.dev)

    def to_boxlists(self, k=0):
        """BoxLists of the LOCAL images from pinned host buffer k (waits for that step's device->host copy only)."""
        from ..structures.bounding_box import BoxList
        self.d2h_done[k].synchronize()
        mine = self.host[k]
        res = []
        for b, (h, w) in enumerate(self.image_sizes):
            n = int(round(float(mine[b, self.max_out, 0])))
            if n > self.max_out:
                raise MqdetError(f"image {b}: {n} detections exceed the {self.max_out}-row result buffer")
            bl = BoxList(mine[b, :n, :4].clone(), (w, h), mode="xyxy")
            bl.add_field("labels", mine[b, :n, 5].long())
            bl.add_field("scores", mine[b, :n, 4].clone())
            res.append(bl)
        return res

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
            yield self.to_boxlists(k)
            if nxt is None:
                return
            k ^= 1


class GroundingDINOEngine:
    """The same idea for ``mqdet_b200.modeling.groundingdino.groundingdino.GroundingDINO`` (BASELINE config 4): the whole forward
    (≈ 780 kernels at 2 images) recorded once as a CUDA graph over a static input buffer and replayed per batch; pinned host images in,
    ``list[BoxList]`` out, and — with ``torch.distributed`` initialised — ONE all-gather of the packed ``[B, num_queries + 1, 6]`` result
    per step (``parallel.all_gather_packed``), issued after the replay, outside the graph.

        eng = GroundingDINOEngine(model, captions, positive_map, batch_shape=(2, 3, 800, 1344), image_sizes=[(800, 1333)] * 2)
        for boxlists in eng.run(host_batches): ...
    """

    def __init__(self, model, captions, positive_map, batch_shape, image_sizes, *, use_graph=True, gather=True, warmup=2):
        self.model, self.captions, self.positive_map = model, captions, positive_map
        self.dev = next(model.parameters()).device
        if self.dev.type != "cuda":
            raise MqdetError("GroundingDINOEngine: the model must live on a CUDA device (no CPU fallback)")
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
        from ..modeling.groundingdino.groundingdino import GroundingDINO
        rank = dist.get_rank() if self.world > 1 else 0
        for hb in host_batches:
            det = self.step_device(hb)
            local = det[rank * self.B:(rank + 1) * self.B] if self.world > 1 else det
            self.host.copy_(local, non_blocking=True)
            torch.cuda.current_stream(self.dev).synchronize()
            yield GroundingDINO.to_boxlists(self.host, self.image_sizes)
