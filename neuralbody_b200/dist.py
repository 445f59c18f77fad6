"""Ray-sharded multi-GPU render (SURVEY.md 8e): rays are independent units, so the rays of every frame are dealt to the
ranks in interleaved chunks (chunk c of `chunk` consecutive rays goes to rank c % world: with exact empty-sample skipping
the cost of a ray depends on how much body it crosses, so contiguous image slabs would be unbalanced), each rank renders
its shard with the fused kernels, and ONE all-gather per frame stitches the image.  No collective runs on the data path
before that.

The reference has no multi-GPU render (run.py:52-69 renders on one device); its only parallelism is DDP over frames in
training (lib/train/trainers/trainer.py:13-18), which is unchanged by this package.

The gathered payload is one fused slab per rank, [rgb(3) | disp | acc | depth] = 24 B/ray, which the render kernels write
directly (nb_render_args.out_ray_stride = 6), so the gather is a single NCCL call (latency-bound: 6.3 MB per 512x512 frame
over NVLink 5 / NVSwitch).  `FrameGatherer` issues it on a side stream with double-buffered slabs, so the gather, the
un-permute and the device->host copy of frame v overlap the render of frame v + 1.
"""
import torch
import torch.distributed as dist

SLAB_KEYS = (("rgb_map", 3), ("disp_map", 1), ("acc_map", 1), ("depth_map", 1))
SLAB_WIDTH = sum(w for _, w in SLAB_KEYS)


def shard_bounds(n_rays, rank, world):
    """Contiguous equal slabs (last ranks may get padding): returns (start, stop, per_rank)."""
    per = (n_rays + world - 1) // world
    start = min(rank * per, n_rays)
    stop = min(start + per, n_rays)
    return start, stop, per


def shard_indices(n_rays, rank, world, chunk=256):
    """Interleaved sharding: ray chunk c (of `chunk` consecutive rays) goes to rank c % world.  Returns (idx, per): idx is a
    LongTensor of `per` ray indices (equal on all ranks; short shards are padded by repeating the last real ray)."""
    n_chunks = (n_rays + chunk - 1) // chunk
    per_chunks = (n_chunks + world - 1) // world
    per = per_chunks * chunk
    mine = torch.arange(rank, n_chunks, world) if rank < n_chunks else torch.zeros(0, dtype=torch.long)
    idx = (mine[:, None] * chunk + torch.arange(chunk)[None, :]).reshape(-1)
    idx = idx[idx < n_rays]
    if idx.numel() < per:
        pad = idx[-1:] if idx.numel() else torch.full((1,), max(n_rays - 1, 0), dtype=torch.long)
        idx = torch.cat([idx, pad.expand(per - idx.numel())])
    return idx, per


_plan_cache = {}


class ShardPlan:
    """The fixed permutation of one (n_rays, world, chunk): which global ray every (rank, local slot) renders, and where every
    global ray sits in the rank-major gathered buffer.  Built once per shape and device and cached (`ShardPlan.get`): nothing
    on the per-frame path touches the host."""

    def __init__(self, n_rays, world, chunk, device):
        self.n_rays, self.world, self.chunk, self.device = int(n_rays), int(world), int(chunk), torch.device(device)
        per = None
        owners = []
        for r in range(world):
            idx, per = shard_indices(n_rays, r, world, chunk)
            owners.append(idx)
        self.per = per
        self.local_index = [o.to(self.device) for o in owners]               # rank -> (per,) global ray of each local slot
        # global ray -> position in the rank-major (world * per) gathered buffer.  A ray rendered twice (padding of a short
        # shard repeats the last real ray) keeps ONE of its copies: they hold equal values.
        src = torch.empty(n_rays, dtype=torch.long)
        flat = torch.cat(owners)
        src[flat] = torch.arange(flat.numel())
        self.gather_index = src.to(self.device)

    @staticmethod
    def get(n_rays, world, chunk=256, device="cpu"):
        key = (int(n_rays), int(world), int(chunk), str(torch.device(device)))
        if key not in _plan_cache:
            _plan_cache[key] = ShardPlan(n_rays, world, chunk, device)
        return _plan_cache[key]

    def shard(self, batch, rank):
        """The per-ray tensors of a reference-style batch dict, restricted to `rank`'s shard (one index_select each)."""
        out = dict(batch)
        idx = self.local_index[rank]
        for k in ("ray_o", "ray_d", "near", "far"):
            out[k] = batch[k].index_select(1, idx.to(batch[k].device))
        return out

    def assemble(self, gathered):
        """(world, B, per, 6) gathered slabs -> (B, n_rays, 6) frame in the original ray order: one index_select."""
        world, B, per, width = gathered.shape
        return gathered.permute(1, 0, 2, 3).reshape(B, world * per, width).index_select(1, self.gather_index.to(gathered.device))


def shard_batch(batch, rank, world, chunk=256):
    """Slice the per-ray tensors of a reference-style batch dict to this rank's interleaved shard."""
    plan = ShardPlan.get(batch["ray_o"].shape[1], world, chunk, batch["ray_o"].device)
    return plan.shard(batch, rank), plan.per


def new_slab(B, per, device):
    """One (B, per, 6) fp32 record per ray + the dict of views the renderer writes through (`Renderer.render_rays(out=...)`)."""
    slab = torch.empty((B, per, SLAB_WIDTH), dtype=torch.float32, device=device)
    return slab, slab_views(slab)


def slab_views(slab):
    out, c = {}, 0
    for k, w in SLAB_KEYS:
        out[k] = slab[..., c:c + w] if w > 1 else slab[..., c]
        c += w
    return out


def pack_slab(ret):
    """dict of dense per-ray outputs (B,nl,*) -> one contiguous (B, nl, 6) fp32 tensor (callers that did not render into a slab)."""
    parts = [ret[k] if w > 1 else ret[k][..., None] for k, w in SLAB_KEYS]
    return torch.cat(parts, dim=-1).contiguous()


def unpack_slab(slab, n_rays, chunk=256):
    """(world, B, per, 6) gathered slabs -> dict of (B, n_rays, *) in the original ray order."""
    plan = ShardPlan.get(n_rays, slab.shape[0], chunk, slab.device)
    return slab_views(plan.assemble(slab))


def gather_slabs(local_slab, group=None, out=None):
    """The one collective of the render path: all_gather_into_tensor of equal-sized slabs."""
    world = dist.get_world_size(group)
    if out is None:
        out = torch.empty((world,) + tuple(local_slab.shape), dtype=local_slab.dtype, device=local_slab.device)
    if local_slab.is_cuda:
        dist.all_gather_into_tensor(out.view(-1), local_slab.reshape(-1), group=group)
    else:  # gloo (CPU tests of the host logic) has no all_gather_into_tensor
        parts = [torch.empty_like(local_slab) for _ in range(world)]
        dist.all_gather(parts, local_slab.contiguous(), group=group)
        out.copy_(torch.stack(parts, 0))
    return out


class FrameGatherer:
    """Double-buffered frame assembly for a stream of ray-sharded views.

        g = FrameGatherer(n_rays, world, rank, device)
        for v in views:
            out = g.begin()                      # dict of slab views for Renderer.render_rays(out=...), compute stream
            renderer.render_rays(..., out=out)   # or, with cfg.render_importance > 0 (coarse + fine sampling):
            #   renderer.render_rays_hierarchical(..., out=out)   -- the fine pass's maps go into the slab
            frame = g.finish()                   # enqueues all-gather + un-permute (+ D2H on rank `host_rank`) on the side stream
        g.drain()                                # frames of the last views are complete after this

    Rays are independent in both passes, so the gathered frame holds the same bits as one unsharded render of the view.

    `finish` returns the (B, n_rays, 6) device frame of THIS view (valid once the side stream has run; `drain` or
    `frame_ready(i).synchronize()`); with `host=True` the view's owner also copies it into a pinned host buffer.  The owner is
    rank `host_rank`, or with `host_rank="rotate"` rank v % world for the v-th view: every GPU then ships 1/world of the frames
    over its own PCIe link instead of rank 0 shipping all of them (8 x 6.3 MB per step at 8 GPUs: 2 ms of a 9 ms step)."""

    def __init__(self, n_rays, world, rank, device, B=1, chunk=256, group=None, host=False, host_rank=0, depth=2):
        self.plan = ShardPlan.get(n_rays, world, chunk, device)
        self.world, self.rank, self.group, self.depth = int(world), int(rank), group, int(depth)
        self.device = torch.device(device)
        self.cuda = self.device.type == "cuda"
        self.side = torch.cuda.Stream(self.device) if self.cuda else None
        per = self.plan.per
        self.slabs = [new_slab(B, per, self.device) for _ in range(depth)]
        self.gathered = [torch.empty((world, B, per, SLAB_WIDTH), dtype=torch.float32, device=self.device) for _ in range(depth)]
        self.frames = [None] * depth
        self.host = None
        self.host_rank = host_rank
        if host and (host_rank == "rotate" or rank == host_rank):
            self.host = [torch.empty((B, n_rays, SLAB_WIDTH), dtype=torch.float32, pin_memory=self.cuda) for _ in range(depth)]
        self.done = [torch.cuda.Event() if self.cuda else None for _ in range(depth)]
        self.v = 0
        self.cur = None

    def begin(self):
        i = self.v % self.depth
        if self.cuda and self.v >= self.depth:
            torch.cuda.current_stream(self.device).wait_event(self.done[i])     # slab i is free again
        self.cur = i
        return self.slabs[i][1]

    def finish(self):
        i = self.cur
        slab = self.slabs[i][0]
        if self.cuda:
            ready = torch.cuda.Event()
            ready.record(torch.cuda.current_stream(self.device))
            with torch.cuda.stream(self.side):
                self.side.wait_event(ready)
                frame = self._assemble(slab, i)
                self.done[i].record(self.side)
        else:
            frame = self._assemble(slab, i)
        self.frames[i] = frame
        self.v += 1
        return frame

    def _assemble(self, slab, i):
        if self.world > 1:
            frame = self.plan.assemble(gather_slabs(slab, self.group, out=self.gathered[i]))
        else:
            frame = self.plan.assemble(slab[None])
        owner = self.v % self.world if self.host_rank == "rotate" else self.host_rank
        if self.host is not None and self.rank == owner:
            self.host[i].copy_(frame, non_blocking=True)
        return frame

    def drain(self):
        if self.cuda:
            self.side.synchronize()


def render_sharded(render_fn, batch, group=None, chunk=256):
    """render_fn(batch) -> dict (e.g. Renderer.render).  Every rank returns the full image dict."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    n = batch["ray_o"].shape[1]
    local, _ = shard_batch(batch, rank, world, chunk)
    ret = render_fn(local)
    gathered = gather_slabs(pack_slab(ret), group)
    return unpack_slab(gathered, n, chunk)
