"""Multi-GPU plumbing: the rasterizer path shards over the batch dimension only (SURVEY.md 8e).

One process per GPU (torchrun); rank r renders samples [lo, hi) of the global batch; there is
no data-path collective.  When a caller needs every image on every rank, `all_gather_images`
performs the single NCCL all-gather named by the north star (gloo on CPU for tests).
"""
import torch
import torch.distributed as dist


def shard_range(batch_size, rank=None, world_size=None):
    """Contiguous shard [lo, hi) of `batch_size` samples owned by `rank`; the first
    batch_size % world_size ranks get one extra sample."""
    if rank is None:
        rank = dist.get_rank() if dist.is_available() and dist.is_initialized() else 0
    if world_size is None:
        world_size = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    if not (0 <= rank < world_size):
        raise ValueError("rank %d outside world of %d" % (rank, world_size))
    base, extra = divmod(batch_size, world_size)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def all_gather_images(images, batch_size=None):
    """Gather per-rank image shards [b_r, ...] into the full batch [B, ...] on every rank.
    Equal shards use one all_gather_into_tensor; ragged shards are padded to the largest."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return images
    world = dist.get_world_size()
    if batch_size is None:
        n = torch.tensor([images.shape[0]], device=images.device)
        sizes = [torch.zeros_like(n) for _ in range(world)]
        dist.all_gather(sizes, n)
        sizes = [int(s.item()) for s in sizes]
    else:
        sizes = [shard_range(batch_size, r, world)[1] - shard_range(batch_size, r, world)[0] for r in range(world)]
    images = images.contiguous()
    if len(set(sizes)) == 1:
        out = torch.empty((sizes[0] * world,) + tuple(images.shape[1:]), dtype=images.dtype, device=images.device)
        dist.all_gather_into_tensor(out, images)
        return out
    mx = max(sizes)
    pad = torch.zeros((mx,) + tuple(images.shape[1:]), dtype=images.dtype, device=images.device)
    pad[:images.shape[0]] = images
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad)
    return torch.cat([p[:s] for p, s in zip(parts, sizes)], dim=0)


class OverlappedImageGather:
    """The optional all-gather of the output images on a side stream, so that it hides behind whatever the caller
    enqueues next (the backward pass; with `chunk` < images_per_rank also the rasterization of the following chunks).

        g = OverlappedImageGather(images_per_rank=4, image_shape=(4, 1024, 1024), device=dev)   # chunk = 4: one push
        img = rasterize(batch)                      # [4, 4, H, W] on the current stream
        g.push(0, img)                              # side stream: wait for img, all-gather it straight into the result
        loss.backward()                             # ... runs while the gather is in flight
        full = g.result()                           # [world * 4, 4, H, W]; the current stream waits for the side stream

    One launch for the whole batch is the fast configuration; chunk = 1 or 2 was slower: a forward launch at this mesh is
    bound by the serial chain of its heaviest blocks however few images it holds, so splitting the batch multiplies that
    (DESIGN.md section 4).

    Sample r * images_per_rank + i of the result is chunk i of rank r, i.e. the same order all_gather_images gives.
    Equal shards only.  On CPU tensors (gloo, tests) the calls run synchronously.  Without a process group the result
    is the concatenation of the local chunks."""

    def __init__(self, images_per_rank, image_shape, device, dtype=torch.float32, chunk=None):
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.n = int(images_per_rank)
        self.chunk = self.n if chunk is None else int(chunk)
        if self.n % self.chunk:
            raise ValueError("images_per_rank %d is not a multiple of chunk %d" % (self.n, self.chunk))
        self.device = torch.device(device)
        self.out = torch.empty((self.world, self.n) + tuple(image_shape), dtype=dtype, device=self.device)
        self.cuda = self.device.type == "cuda"
        self.side = torch.cuda.Stream(self.device) if self.cuda else None
        # chunk == images_per_rank: the gather lands in `out` directly; smaller chunks go through a rank-major staging
        # block each and are placed into their column of the [world, images_per_rank] result on the side stream
        self.tmp = [torch.empty((self.world * self.chunk,) + tuple(image_shape), dtype=dtype, device=self.device)
                    for _ in range(self.n // self.chunk)] if (self.world > 1 and self.chunk != self.n) else None
        self._keep = []   # the pushed images stay referenced until result(): the side stream reads them

    def push(self, index, images):
        """images: chunk number `index` of this rank, [chunk, *image_shape], produced on the current stream."""
        lo = index * self.chunk
        images = images.detach()
        if self.world == 1:
            self.out[0, lo:lo + self.chunk].copy_(images)
            return
        src = images.contiguous()
        dst = self.tmp[index] if self.tmp is not None else self.out.view((self.world * self.n,) + tuple(self.out.shape[2:]))
        if not self.cuda:
            dist.all_gather_into_tensor(dst, src)
            if self.tmp is not None:
                self.out[:, lo:lo + self.chunk].copy_(dst.view((self.world, self.chunk) + tuple(self.out.shape[2:])))
            return
        # No Tensor.record_stream here: a recorded block makes the caching allocator poll events on every later
        # allocation and grow the pool while they are pending (measured: the C3 step took about three times as long).  Holding
        # the reference until result() -- after which the current stream has waited for the side stream -- is enough.
        self._keep.append(src)
        self.side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.side):
            dist.all_gather_into_tensor(dst, src)
            if self.tmp is not None:
                self.out[:, lo:lo + self.chunk].copy_(dst.view((self.world, self.chunk) + tuple(self.out.shape[2:])))

    def result(self):
        if self.cuda and self.world > 1:
            torch.cuda.current_stream(self.device).wait_stream(self.side)
        self._keep.clear()
        return self.out.view((self.world * self.n,) + tuple(self.out.shape[2:]))
