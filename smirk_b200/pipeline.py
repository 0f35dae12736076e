"""``SmirkPipeline`` — the whole per-frame hot path as one call: encode -> FLAME -> render (-> generator).

This is the public entry point ``bench.py`` and the demos use for batched work:

* ``forward(img)``            device tensors in, dict of device tensors out (what demo.py:107-112 does
                              with three module calls);
* ``capture(B)`` / ``replay`` the same work recorded once into a CUDA graph (one launch per batch instead
                              of ~100 kernel launches — the launch-bound regime of small batches);
* ``submit(i, img)`` / ``join`` software pipelining over ``slots`` lanes: each lane owns a replica of the
                              modules (same weights, its own native handles, workspaces, graph and stream),
                              so the serial FLAME -> rasteriser tail of batch i overlaps the encoder of
                              batch i+1;
* ``run_host(img_pinned, i)`` end-to-end from pinned host memory: H2D copy, graph replay, D2H of the
                              results into pinned buffers; lane i % slots, copies on a second stream, so
                              the copies of one batch overlap the kernels of the other;
* ``shard_bounds`` / ``all_gather_frames``  frame-shard data parallelism (one process per GPU, contiguous
                              split of the batch; a single NCCL all-gather of the final outputs — SURVEY.md §8e);
* ``video=VideoStage(...)``  uint8 frames in, the video demo's output grid out (``smirk_b200.video``): the batch's
                              crop, the hot path and the grid in one call / one graph; the auxiliary input is the
                              ``VideoBatch`` of ``VideoStage.prepare``;
* ``enable_gather(keys)``     puts that all-gather INTO the pipeline: after every batch the lane's outputs are gathered
                              over all ranks on a communication stream (NCCL over NVLink / NVSwitch), overlapping the
                              kernels of the next batches on the other lanes.

Captured graphs snapshot the packed weights and workspaces they were recorded with and keep them alive
(``rec["keep"]``); after changing weights, ``precision`` or devices call ``refresh()`` to re-capture.
"""
import copy

import torch

from . import _lib


def shard_bounds(n_frames, world_size, rank):
    """Contiguous split of ``n_frames`` over ``world_size`` ranks (SURVEY.md §8e): rank g owns
    [lo, hi).  The first ``n_frames % world_size`` ranks take one extra frame."""
    base, rem = divmod(n_frames, world_size)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def all_gather_frames(t, n_frames=None, group=None):
    """Gather per-rank frame shards (dim 0) into the full batch on every rank.  Ragged shards are padded
    to the largest shard for one equal-count ``all_gather_into_tensor`` and trimmed afterwards."""
    import torch.distributed as dist
    ws = dist.get_world_size(group)
    if ws == 1:
        return t
    counts = [shard_bounds(n_frames, ws, r)[1] - shard_bounds(n_frames, ws, r)[0] for r in range(ws)] \
        if n_frames is not None else [t.shape[0]] * ws
    mx = max(counts)
    if t.shape[0] < mx:
        pad = torch.zeros((mx - t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
        t = torch.cat([t, pad], 0)
    out = torch.empty((ws * mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    dist.all_gather_into_tensor(out, t.contiguous(), group=group)
    if all(c == mx for c in counts):
        return out
    return torch.cat([out[r * mx:r * mx + c] for r, c in enumerate(counts)], 0)


class _Lane:
    """One pipeline lane: a set of modules, a compute stream, a copy stream, per-batch-size graphs."""

    def __init__(self, modules, device, own_stream):
        self.encoder, self.flame, self.renderer, self.generator, self.masking, self.video = modules
        self.stream = torch.cuda.Stream(device=device) if own_stream else None
        self.graphs = {}
        self.host = {}
        self.computed = torch.cuda.Event()
        self.done = torch.cuda.Event()
        self.staged = torch.cuda.Event()
        self.consumed = torch.cuda.Event()
        self.gathered = torch.cuda.Event()
        self.gather_out = {}

    def modules(self):
        return [m for m in (self.encoder, self.flame, self.renderer, self.generator, self.masking, self.video) if m is not None]


class _PeerBuffer:
    """One rank's gather buffer of one lane, allocated by the native library (``smk_peer_alloc``: a plain cudaMalloc whose
    CUDA IPC handle other ranks can open) plus this rank's mappings of every peer's buffer.  ``local`` is a uint8 tensor view
    of the own buffer, ``ptrs[r]`` the device address of rank r's buffer as seen from this process."""

    def __init__(self, nbytes, device):
        import ctypes as C
        ptr, handle = C.c_void_p(), C.create_string_buffer(64)
        _lib.call("smk_peer_alloc", device, nbytes, C.byref(ptr), handle)
        self.ptr, self.nbytes, self.handle, self.ptrs, self._mapped = ptr.value, nbytes, handle.raw, [], []
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (self.ptr, False), "version": 2}
        self.local = torch.as_tensor(self, device=device)

    def map_peers(self, handles, rank, shard, offsets=(0,)):
        """Open every peer's handle; ``dsts[j]`` = where part j (byte offset ``offsets[j]``) of this rank's shard goes in each
        PEER's buffer (slot ``rank``), starting with the next rank.  The own slot is not a destination: see ``SmirkPipeline.gathered``."""
        import ctypes as C
        for r, h in enumerate(handles):
            if r == rank:
                self.ptrs.append(self.ptr)
                continue
            p = C.c_void_p()
            _lib.call("smk_peer_open", self.local.device, h, C.byref(p))
            self._mapped.append(p.value)
            self.ptrs.append(p.value)
        self.local = self.local.view(len(handles), -1)
        ws = len(handles)
        self.dsts = [(C.c_void_p * (ws - 1))(*[self.ptrs[(rank + 1 + d) % ws] + rank * shard + off for d in range(ws - 1)]) for off in offsets]

    def __del__(self):
        # Only this process's mappings of the PEERS' buffers are closed here.  The own buffer is exported: CUDA leaves freeing
        # it while another process may still have it mapped undefined, and a destructor cannot synchronise with the peers, so
        # it is left to process teardown (a gather set-up is made once per pipeline; bench.py's two pipelines hold 0.7 + 5.9 GB
        # at 8 GPUs).  A host that re-creates pipelines can call smk_peer_free itself after a barrier.
        try:
            for p in self._mapped:
                _lib.call("smk_peer_close", self.local.device, p)
            self._mapped = []
        except Exception:
            pass


class SmirkPipeline:
    OUT_KEYS = ("rendered_img", "vertices", "transformed_vertices", "landmarks_fan", "landmarks_mp", "params")

    def __init__(self, encoder, flame, renderer, generator=None, device="cuda:0", slots=2, masking=None, video=None):
        """``masking``: a ``smirk_b200.masking.MaskingStage``.  With it the full cycle computes the generator's second
        input itself (demo.py:138-165) and the auxiliary input of forward/replay/submit/run_host is the landmark hull mask
        [B,1,224,224]; without it the auxiliary input is a ready-made ``masked_img`` [B,3,224,224].
        ``video``: a ``smirk_b200.video.VideoStage``.  With it the first input of forward/replay/submit/run_host is a
        batch of uint8 BGR frames [B,H,W,3], the auxiliary input the ``VideoBatch`` of ``video.prepare``, and the outputs
        gain ``cropped_img`` and ``grid`` (and, with a generator, ``hull_mask``; the generator then needs ``masking``)."""
        if video is not None and generator is not None and masking is None:
            raise ValueError("SmirkPipeline: the video stage's generator panel needs masking=MaskingStage(...) "
                             "(the hull mask goes through the masking step, demo_video.py:177-197)")
        self.device = torch.device(device)
        self.encoder, self.flame, self.renderer, self.generator, self.masking = encoder, flame, renderer, generator, masking
        self.video = video
        self.slots = max(1, int(slots))
        self._lanes = [_Lane(self._modules(), self.device, own_stream=False)]
        self._h2d = self._d2h = None
        self._gather_keys, self._gather_group, self._comm, self._gather_backend, self._p2p = (), None, None, None, None

    def _modules(self):
        return (self.encoder, self.flame, self.renderer, self.generator, self.masking, self.video)

    def refresh(self):
        """Drop every captured graph (and the weights / workspaces they kept alive) and the lane replicas, so the next
        call re-captures from the current state of the caller's modules."""
        torch.cuda.synchronize(self.device)
        self._lanes = [_Lane(self._modules(), self.device, own_stream=False)]

    def _lane(self, i):
        """Lane 0 runs the caller's modules on the caller's stream; lanes >= 1 are replicas (deep copies:
        same parameter values, separate native handles / workspaces) on their own streams."""
        while len(self._lanes) <= i:
            mods = tuple(copy.deepcopy(m) if m is not None else None for m in self._modules())
            self._lanes.append(_Lane(mods, self.device, own_stream=True))
        return self._lanes[i]

    # ---- plain forward (device in, device out) -----------------------------------------------------
    @torch.no_grad()
    def forward(self, img, masked_img=None, lane=0):
        if self.video is not None:                  # img = uint8 frames, masked_img = the VideoBatch
            self._check_video(img, masked_img)
            aux = [masked_img[k].to(img.device, non_blocking=True) for k in self._video_keys()]
            return self._forward_video(img, aux, lane)
        return self._forward(self._lane(lane), img, masked_img)

    def _forward_video(self, frames, aux, lane):
        """Crop (or resize), the hot path, the output grid (smirk_b200/video.py); aux = the device tensors of
        ``_video_keys()``, in that order: crop / back matrices [B,9] with the crop, the int32 landmarks [B,L,2] with a
        generator."""
        L = self._lane(lane)
        aux = dict(zip(self._video_keys(), aux))
        img = L.video.crop(frames, aux.get("crop_m"))
        hull = L.video.hull_mask(aux["kpt"]) if L.generator is not None else None
        out = self._forward(L, img, hull)
        out["cropped_img"] = img
        panels = [out["rendered_img"]]
        if hull is not None:
            out["hull_mask"] = hull
            panels.append(out["reconstructed_img"])
        out["grid"] = L.video.compose(frames, img, panels, aux.get("back_m"))
        return out

    def _video_keys(self):
        keys = ("crop_m", "back_m") if self.video.use_crop else ()
        return keys + ("kpt",) if self.generator is not None else keys

    def _check_video(self, frames, batch):
        self.video.check(frames, batch)
        missing = [k for k in self._video_keys() if k not in batch]
        if missing:
            raise ValueError("SmirkPipeline: the VideoBatch lacks %s (the generator's hull mask needs the landmarks: "
                             "VideoStage.prepare(landmarks))" % ", ".join(missing))

    def _forward(self, L, img, masked_img):
        p = L.encoder(img)
        fo = L.flame.forward(p)
        ro = L.renderer.forward(fo["vertices"], p["cam"], landmarks_fan=fo["landmarks_fan"],
                                landmarks_mp=fo["landmarks_mp"])
        out = {
            "rendered_img": ro["rendered_img"], "vertices": fo["vertices"],
            "transformed_vertices": ro["transformed_vertices"], "landmarks_fan": ro["landmarks_fan"],
            "landmarks_mp": ro["landmarks_mp"],
            "params": torch.cat([p["pose_params"], p["cam"], p["shape_params"], p["expression_params"],
                                 p["eyelid_params"], p["jaw_params"]], 1),                      # [B,361]
        }
        if L.generator is not None:
            if masked_img is None:
                raise RuntimeError("SmirkPipeline: the generator stage needs `masked_img` (demo.py:165-167), or the hull mask "
                                   "when a MaskingStage is attached")
            if L.masking is not None:           # the auxiliary input is the hull mask: demo.py:138-165 on the device
                masked_img = L.masking(img, masked_img, ro["transformed_vertices"], ro["rendered_img"])
                out["masked_img"] = masked_img
            out["reconstructed_img"] = L.generator(torch.cat([ro["rendered_img"], masked_img], 1))
        return out

    # ---- CUDA graph -----------------------------------------------------------------------------------
    def capture(self, B, lane=0):
        """Record forward() for batch size B into a CUDA graph with static input/output buffers."""
        L = self._lane(lane)
        if B in L.graphs:
            return L.graphs[B]
        dev = self.device
        static_aux = []
        static_mask = None                                  # the video stage draws its hull mask inside the graph
        if self.generator is not None and self.video is None:
            static_mask = torch.zeros(B, 1 if self.masking is not None else 3, 224, 224, device=dev)
        if self.video is not None:                          # frames + the tensors of the VideoBatch
            static_in = torch.zeros((B,) + self.video.frame_hw + (3,), dtype=torch.uint8, device=dev)
            shapes = {"crop_m": ((B, 9), torch.float64), "back_m": ((B, 9), torch.float64),
                      "kpt": ((B, self.video.L, 2), torch.int32)}
            static_aux = [torch.zeros(shapes[k][0], dtype=shapes[k][1], device=dev) for k in self._video_keys()]
            run = lambda: self._forward_video(static_in, static_aux, lane)
        else:
            static_in = torch.zeros(B, 3, 224, 224, device=dev)
            run = lambda: self.forward(static_in, static_mask, lane)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):                       # warm-up: builds handles, sizes workspaces
            for _ in range(2):
                run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        n0 = _lib.call("smk_launch_count", dev)
        with torch.cuda.graph(g):
            static_out = run()
        launches = _lib.call("smk_launch_count", dev) - n0
        # The graph holds raw pointers into each module's packed weights (native handle) and workspace: keep both
        # alive for as long as the graph exists, whatever the modules do afterwards (re-pack, grow their workspace
        # for a larger batch, ...).  A workspace that grows allocates a NEW buffer, so graphs of different batch
        # sizes on one lane never alias a freed one.
        keep = [m.graph_keep_alive() for m in L.modules()]
        rec = dict(graph=g, img=static_in, mask=static_mask, aux=static_aux, out=static_out, launches=int(launches), keep=keep)
        L.graphs[B] = rec
        return rec

    def replay(self, img, masked_img=None):
        """Lane 0, caller's stream: copy the inputs into the graph's static buffers and replay."""
        if self.video is not None:
            self._check_video(img, masked_img)
        rec = self.capture(img.shape[0])
        rec["img"].copy_(img, non_blocking=True)
        if rec["mask"] is not None:
            rec["mask"].copy_(masked_img, non_blocking=True)
        self._copy_aux(rec["aux"], self._upload_aux(masked_img, torch.cuda.current_stream(self.device)))
        rec["graph"].replay()
        return rec["out"]

    # ---- software pipelining over lanes -------------------------------------------------------------
    def submit(self, i, img, masked_img=None):
        """Enqueue batch ``i`` on lane ``i % slots`` (its own stream; lane 0 = the caller's stream).  Inputs
        must already be valid on the caller's current stream.  Outputs live in the lane's static buffers
        until that lane is used again; call ``join()`` before reading them from the caller's stream."""
        lane = i % self.slots
        if self.video is not None:
            self._check_video(img, masked_img)
        rec = self.capture(img.shape[0], lane)
        L = self._lanes[lane]
        cur = torch.cuda.current_stream(self.device)
        if L.stream is None:
            if self._gather_keys:
                cur.wait_event(L.gathered)
            self.replay(img, masked_img)
            L.computed.record(cur)
            self._gather(L, rec)
            return rec["out"]
        L.stream.wait_stream(cur)                           # inputs ready
        aux = self._upload_aux(masked_img, L.stream)
        with torch.cuda.stream(L.stream):
            if self._gather_keys:
                L.stream.wait_event(L.gathered)             # the previous all-gather of this lane has read the outputs
            rec["img"].copy_(img, non_blocking=True)
            if rec["mask"] is not None:
                rec["mask"].copy_(masked_img, non_blocking=True)
            self._copy_aux(rec["aux"], aux)
            rec["graph"].replay()
            L.computed.record(L.stream)
        self._gather(L, rec)
        return rec["out"]

    def _upload_aux(self, batch, consumer):
        """The video stage's graph inputs besides the frames (``_video_keys()`` of a VideoBatch), on the device and valid on
        ``consumer``: host tensors are uploaded on the H2D stream, device tensors are used as they are.  None without the
        video stage."""
        if self.video is None:
            return None
        src = [batch[k] for k in self._video_keys()]
        if all(t.is_cuda for t in src):
            return src
        if self._h2d is None:
            self._h2d, self._d2h = torch.cuda.Stream(device=self.device), torch.cuda.Stream(device=self.device)
        with torch.cuda.stream(self._h2d):
            dev = [t.to(self.device, non_blocking=True) for t in src]
        consumer.wait_stream(self._h2d)
        for t in dev:
            t.record_stream(consumer)
        return dev

    @staticmethod
    def _copy_aux(static_aux, src):
        """Copy the video stage's graph inputs (a list of device tensors) into the graph's static buffers."""
        for s, t in zip(static_aux, src or ()):
            s.copy_(t, non_blocking=True)

    # ---- all-gather of the final outputs inside the pipeline (frame-shard data parallelism) ----------------
    def enable_gather(self, keys=("rendered_img", "vertices", "params"), group=None, backend="auto"):
        """After every batch, all-gather the listed outputs over the process group (dim 0 = rank-major frames) on a
        communication stream; results land in ``gathered(i, key)``.  ``keys = ()`` switches it off.

        backend "p2p" (= "auto" when every rank can map its peers): each rank owns one gather buffer per lane, maps every
        peer's buffer once (CUDA IPC, ``smk_peer_*`` in the C ABI) and after a batch PUSHES every output into slot ``rank``
        of every peer's buffer with copy-engine copies (csrc/peer.cu; directly from the output tensors with one peer, packed
        first with more: see ``_gather``) — no SM is taken from the persistent compute kernels, and the own shard stays in the
        output tensor until ``gathered()`` is called.  A slot of
        a peer's buffer is rewritten ``slots`` batches later; ``gather_sync()`` (stream join + group barrier) makes a batch's
        gathered tensors safe to read.
        backend "nccl": ``all_gather_into_tensor`` over NVLink / NVSwitch.  NCCL's kernels occupy SMs while the compute
        kernels (one persistent CTA per SM each) run, which splits every overlapped launch into two waves."""
        import torch.distributed as dist
        self._gather_keys = tuple(keys) if (dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1) else ()
        self._gather_group = group
        self._gather_backend = None
        if self._gather_keys:
            if self._comm is None:
                self._comm = torch.cuda.Stream(device=self.device)
            self._gather_backend = "nccl" if backend == "nccl" else "pending-" + backend
        return self._gather_keys

    def _setup_p2p(self, B):
        """Allocate one packed gather buffer per lane ([world, bytes of one shard]) and map every peer's buffers (CUDA IPC).
        Collective: every rank must call it with the same B.  Returns True when every rank succeeded."""
        import torch.distributed as dist
        ws, rank = dist.get_world_size(self._gather_group), dist.get_rank(self._gather_group)
        ok, sizes, offsets, shard, mine, bufs = True, [], [], 0, None, []
        pack = ws > 2
        try:
            rec = self.capture(B)
            assert all(rec["out"][k].is_contiguous() for k in self._gather_keys)
            sizes = [rec["out"][k].numel() * rec["out"][k].element_size() for k in self._gather_keys]
            offsets = [sum((m + 255) // 256 * 256 for m in sizes[:j]) for j in range(len(sizes))]
            shard = sum((n + 255) // 256 * 256 for n in sizes)
            with torch.cuda.device(self.device):
                bufs = [_PeerBuffer(ws * shard, self.device) for _ in range(self.slots)]
            mine = [b.handle for b in bufs]
        except Exception:
            ok, mine = False, None
        everyone = [None] * ws
        dist.all_gather_object(everyone, mine, group=self._gather_group)
        ok = ok and all(e is not None for e in everyone)
        if ok:
            try:
                with torch.cuda.device(self.device):
                    for lane in range(self.slots):
                        L = self._lane(lane)
                        L.p2p = bufs[lane]
                        L.p2p.map_peers([everyone[r][lane] for r in range(ws)], rank, shard, offsets)
                        L.p2p_stage = torch.empty(shard, dtype=torch.uint8, device=self.device) if pack else None
                    import ctypes as C
                    fan = C.c_void_p()
                    _lib.call("smk_peer_fan_create", self.device, min(ws, 8), C.byref(fan))
                    self._fan = _lib.NativeHandle(fan, "smk_peer_fan_destroy")
                torch.cuda.synchronize(self.device)
            except Exception:
                ok = False
        flag = torch.tensor([1 if ok else 0], device=self.device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self._gather_group)
        ok = bool(flag.item())
        self._p2p = dict(B=B, sizes=sizes, offsets=offsets, shard=shard, rank=rank, pack=pack) if ok else None
        return ok

    def _gather(self, L, rec):
        if not self._gather_keys:
            return
        import torch.distributed as dist
        ws = dist.get_world_size(self._gather_group)
        B = rec["img"].shape[0]
        if self._gather_backend.startswith("pending-"):
            want = self._gather_backend[8:]
            self._gather_backend = "p2p" if (want in ("auto", "p2p") and self._setup_p2p(B)) else "nccl"
        if self._gather_backend == "p2p" and self._p2p["B"] != B:
            self._gather_backend = "p2p" if self._setup_p2p(B) else "nccl"
        if self._gather_backend == "p2p":
            # Copy-engine copies into slot `rank` of each PEER's buffer on the fan's streams; the own shard is never copied.
            #   direct (one peer): every output goes from where the kernels wrote it, one copy per (output, peer) — device-local
            #     copies are what hurts the concurrent compute kernels (tools/bench_peer_load.py measures it), so none is made.
            #   packed (more peers): the outputs are first packed into one staging buffer and each peer gets ONE copy instead of
            #     one per (output, peer).
            with torch.cuda.stream(self._comm):
                self._comm.wait_event(L.computed)
                if self._p2p["pack"]:
                    for k, n, off in zip(self._gather_keys, self._p2p["sizes"], self._p2p["offsets"]):
                        L.p2p_stage[off:off + n].copy_(rec["out"][k].reshape(-1).view(torch.uint8), non_blocking=True)
                    # The lane may overwrite its outputs as soon as they are PACKED: the pushes read the staging buffer only, and
                    # its reuse is ordered by this stream (a fan push ends with the stream waiting for every copy).  Releasing
                    # the lane after the pushes instead idles it for their whole duration.
                    L.gathered.record(self._comm)
                    _lib.call("smk_peer_fan_push", self.device, self._fan, L.p2p.dsts[0], ws - 1, L.p2p_stage, self._p2p["shard"])
                else:
                    for j, (k, n) in enumerate(zip(self._gather_keys, self._p2p["sizes"])):
                        _lib.call("smk_peer_fan_push", self.device, self._fan, L.p2p.dsts[j], ws - 1, rec["out"][k], n)
                    L.gathered.record(self._comm)
            return
        with torch.cuda.stream(self._comm):
            self._comm.wait_event(L.computed)
            for k in self._gather_keys:
                t = rec["out"][k]
                key = (k, tuple(t.shape))
                if key not in L.gather_out:
                    L.gather_out[key] = torch.empty((ws * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
                dist.all_gather_into_tensor(L.gather_out[key], t, group=self._gather_group)
            L.gathered.record(self._comm)

    def gather_sync(self):
        """Make the gathered tensors of every submitted batch readable: join the streams, then (p2p) a group barrier so that
        every peer's pushes into this rank's buffers have landed."""
        import torch.distributed as dist
        self.join()
        torch.cuda.synchronize(self.device)
        if self._gather_keys and self._gather_backend == "p2p":
            dist.barrier(group=self._gather_group)

    def gathered(self, i, key):
        """The all-gathered ``key`` of the batch last submitted on lane ``i % slots`` (valid after ``gather_sync()``)."""
        L = self._lanes[i % self.slots]
        if self._gather_backend == "p2p":
            rec = L.graphs[self._p2p["B"]]
            j = self._gather_keys.index(key)
            off, n, t = self._p2p["offsets"][j], self._p2p["sizes"][j], rec["out"][key]
            # the own shard was never copied: it still sits in the pipeline's output tensor and joins the peers' shards here
            L.p2p.local[self._p2p["rank"], off:off + n].copy_(t.reshape(-1).view(torch.uint8))
            return L.p2p.local[:, off:off + n].contiguous().view(t.dtype).reshape((-1,) + tuple(t.shape[1:]))
        for (k, _), v in L.gather_out.items():
            if k == key:
                return v
        raise KeyError(key)

    def gather_bytes_per_step(self, B):
        """Bytes this rank RECEIVES per step in the all-gather ((world_size - 1) shards; it sends as many)."""
        if not self._gather_keys:
            return 0
        import torch.distributed as dist
        rec = self.capture(B)
        return (dist.get_world_size(self._gather_group) - 1) * sum(rec["out"][k].numel() * rec["out"][k].element_size() for k in self._gather_keys)

    def join(self):
        cur = torch.cuda.current_stream(self.device)
        for L in self._lanes:
            if L.stream is not None:
                cur.wait_stream(L.stream)
        for st in (getattr(self, "_h2d", None), getattr(self, "_d2h", None), getattr(self, "_comm", None)):
            if st is not None:
                cur.wait_stream(st)

    # ---- host-to-host (pinned) ------------------------------------------------------------------------
    def host_buffers(self, B, lane, keys=("rendered_img", "vertices", "params")):
        """Per-lane pinned output buffers + device staging buffers; one H2D and one D2H stream for the whole
        pipeline (copies in one direction serialise on the link anyway)."""
        L = self._lane(lane)
        key = (B, tuple(keys))
        if key not in L.host:
            rec = self.capture(B, lane)
            L.host[key] = dict(
                out={k: torch.empty(rec["out"][k].shape, dtype=rec["out"][k].dtype).pin_memory() for k in keys},
                dev_in=torch.empty_like(rec["img"]),
                dev_mask=torch.empty_like(rec["mask"]) if rec["mask"] is not None else None,
                dev_aux=[torch.empty_like(a) for a in rec["aux"]],
                dev_out={k: torch.empty_like(rec["out"][k]) for k in keys})
            if getattr(self, "_h2d", None) is None:
                self._h2d = torch.cuda.Stream(device=self.device)
                self._d2h = torch.cuda.Stream(device=self.device)
        return L.host[key]

    def run_host(self, img_pinned, i, masked_pinned=None, keys=("rendered_img", "vertices", "params")):
        """Batch ``i``, host to host, three decoupled stages:
          H2D stream   pinned images -> the lane's device staging buffer (as soon as that buffer is free);
          lane stream  staging -> graph input, graph replay, graph outputs -> output staging;
          D2H stream   output staging -> the lane's pinned result buffers.
        With ``slots`` lanes the upload of batch i+1 and the download of batch i-1 overlap the kernels of
        batch i.  Returns the lane's pinned output dict — ``join()`` (or ``lane_done(i).synchronize()``)
        before reading it."""
        B = img_pinned.shape[0]
        if self.video is not None:
            self._check_video(img_pinned, masked_pinned)
        lane = i % self.slots
        hb = self.host_buffers(B, lane, keys)
        rec = self.capture(B, lane)
        L = self._lanes[lane]
        cur = torch.cuda.current_stream(self.device)
        compute = L.stream if L.stream is not None else cur
        with torch.cuda.stream(self._h2d):
            self._h2d.wait_event(L.consumed)                # staging input of this lane has been read by its previous batch
            hb["dev_in"].copy_(img_pinned, non_blocking=True)
            if hb["dev_mask"] is not None:
                hb["dev_mask"].copy_(masked_pinned, non_blocking=True)
            if hb["dev_aux"]:
                self._copy_aux(hb["dev_aux"], [masked_pinned[k] for k in self._video_keys()])
            L.staged.record(self._h2d)
        with torch.cuda.stream(compute):
            compute.wait_event(L.staged)
            compute.wait_event(L.done)                      # output staging drained by the previous D2H of this lane
            if self._gather_keys:
                compute.wait_event(L.gathered)
            rec["img"].copy_(hb["dev_in"], non_blocking=True)
            if rec["mask"] is not None:
                rec["mask"].copy_(hb["dev_mask"], non_blocking=True)
            self._copy_aux(rec["aux"], hb["dev_aux"])
            L.consumed.record(compute)
            rec["graph"].replay()
            for k in keys:
                hb["dev_out"][k].copy_(rec["out"][k], non_blocking=True)
            L.computed.record(compute)
        self._gather(L, rec)
        with torch.cuda.stream(self._d2h):
            self._d2h.wait_event(L.computed)
            for k in keys:
                hb["out"][k].copy_(hb["dev_out"][k], non_blocking=True)
            L.done.record(self._d2h)
        return hb["out"]

    def lane_done(self, i):
        return self._lanes[i % self.slots].done

    def bytes_per_step(self, B, keys=("rendered_img", "vertices", "params")):
        rec = self.capture(B)
        h2d = B * 3 * 224 * 224 * 4 + (rec["mask"].numel() * 4 if rec["mask"] is not None else 0)
        if self.video is not None:
            h2d = sum(t.numel() * t.element_size() for t in [rec["img"]] + rec["aux"])
        d2h = sum(rec["out"][k].numel() * rec["out"][k].element_size() for k in keys)
        return h2d, d2h

    def launches_per_step(self, B):
        return self.capture(B)["launches"]
