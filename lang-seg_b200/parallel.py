"""Multi-GPU host logic: one process per GPU, batch sharded, one collective (SURVEY.md section 8(e)).

The image path has no cross-image operation in eval mode (BatchNorm uses running statistics), so the
batch shards across ranks with NO data-path collective; weights are resident per rank and text features
are computed redundantly per rank (150 KB, cheaper than a broadcast). The only exchange is the gather of
the final logits: an NCCL all-gather over NVLink / NVSwitch (gloo in the CPU tests).
This replaces the reference's single-process, thread-per-GPU DataParallel with a per-call parameter
broadcast (additional_utils/models.py:35-53,183-248).
"""
import torch
import torch.distributed as dist


def shard_bounds(batch, rank, world):
    """Contiguous shard [lo, hi) of a batch of `batch` images for `rank` (remainder to the low ranks)."""
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def shard_batch(x, rank=None, world=None):
    rank = dist.get_rank() if rank is None else rank
    world = dist.get_world_size() if world is None else world
    lo, hi = shard_bounds(x.shape[0], rank, world)
    return x[lo:hi]


def gather_logits(local, batch=None, group=None):
    """All-gather per-rank logits [b_r, K, H, W] into [sum b_r, K, H, W] in rank order on every rank.
    Equal shards use a single all_gather_into_tensor (in-place receive); ragged shards pad to the max."""
    world = dist.get_world_size(group)
    if world == 1:
        return local
    sizes = [torch.zeros(1, dtype=torch.int64, device=local.device) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([local.shape[0]], dtype=torch.int64, device=local.device), group=group)
    sizes = [int(s.item()) for s in sizes]
    if len(set(sizes)) == 1:
        out = torch.empty((world * sizes[0],) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    mx = max(sizes)
    padded = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    padded[: local.shape[0]] = local
    bufs = [torch.empty_like(padded) for _ in range(world)]
    dist.all_gather(bufs, padded, group=group)
    return torch.cat([b[:s] for b, s in zip(bufs, sizes)], dim=0)


def forward_sharded(net, x_global, labelset=""):
    """Each rank runs net.forward on its contiguous shard of the global batch and gathers the logits. A rank whose shard
    is empty (batch < world size) contributes an empty [0,K,H,W] tensor instead of calling the engine (which rejects
    B = 0), so the collective is still entered by everybody."""
    local = shard_batch(x_global)
    if local.shape[0] == 0:
        k = len(labelset) if not isinstance(labelset, (str, torch.Tensor)) else (
            labelset.shape[0] if isinstance(labelset, torch.Tensor) else len(net.labels))
        out = torch.empty((0, k) + tuple(x_global.shape[2:]), dtype=torch.float32, device=x_global.device)
    else:
        out = net(local.contiguous(), labelset) if not (isinstance(labelset, str) and labelset == "") else net(
            local.contiguous())
    return gather_logits(out)


# ---------------------------------------------------------------------------------------------------------------------
# The bench / serving gather: every step's logits of all ranks end up on `root` as fp32 [world*B, K, H, W].
# ---------------------------------------------------------------------------------------------------------------------
_FLAG_BYTES = 4096        # per-rank flag page at the head of the IPC buffer: uint64 flags
_CONSUMED = 64            # flag index "root has consumed step s" (in every rank's OWN page, written by root)


class LogitsGather:
    """Per-step logits gather to `root` with the bytes the path actually has to move.

    What crosses NVLink is the reference's fp16 matmul result [B,K,H/2,W/2] (lseg_net.py:194-196), 1/8 of the fp32
    [B,K,H,W] logits it determines; `root` runs the x2 align_corners upsample (lseg_net.py:203, lseg_upsample2x_nchw —
    bit-identical to what each rank would have produced) over all world*B*K gathered planes on a side stream, so it
    overlaps the next step's compute. Per step:
        rank r   : forward_lowres -> [comm stream] wait(root consumed step s-2) -> copy-engine push into root's slot
                   (s & 1, r) over NVLink -> release-flag ready[r] = s in root memory
        root     : forward_lowres into its own slot -> [comm stream] acquire ready[1..] >= s -> upsample all slots ->
                   release-flag consumed = s in every peer's memory
    Everything is enqueued on CUDA streams; there is no host synchronisation and no NCCL call on the data path.
    modes: "p2p_copy" (default, above); "p2p_store" — the pixel x text GEMM's epilogue stores straight into root's slot
    (no local copy; the stores contend on root's NVLink ingress when many ranks finish together); "nccl" — all-gather
    of the fp16 low-res logits through torch.distributed, then the same root-side upsample (fallback when CUDA IPC is not
    available; also what the gloo CPU tests exercise).
    """

    def __init__(self, engine, B, K, H, W, root=0, mode="p2p_copy", group=None, timeout_ms=30000, materialize=True,
                 background=False, pipelined=False):
        self.engine, self.B, self.K, self.H, self.W = engine, B, K, H, W
        self.background = background
        # pipelined=True (p2p modes): the gathering rank expands step s-1 on its MAIN stream right after its own forward of
        # step s, instead of expanding step s on a side stream while the trunk of step s+1 runs. The expansion cannot
        # overlap the trunk anyway (it needs the SMs the trunk's CTAs fill); interleaved with it, it costs more than its
        # own time (N = 8: 11.0 ms/step against 8.4 + 1.8), and the data of step s-1 has long arrived, so nothing waits.
        # forward() then returns the gathered logits of the PREVIOUS step (None at the first call); flush() the last.
        self.pipelined = pipelined and mode.startswith("p2p")
        self._expanded = 0
        self.repeat = 1  # tools/gather_check.py --root-repeat: emulate the expansion load of a larger world
        # images the gathering rank computes itself (<= B). It also expands every shard to fp32 (~29 us per image of
        # HBM writes that cannot overlap its trunk), so with equal shards it is the slowest rank; `root_batch` < B
        # balances that (bench.py `gather.balanced`). Its slot keeps B entries; entries >= root_batch are not written.
        self.root_batch = B
        # materialize=False: root keeps the gathered fp16 low-res logits (`lowres()`), the exact information content of
        # the step, and does not expand them to fp32 — what a consumer that takes the argmax / a crop would want
        self.materialize = materialize
        self.group, self.root, self.timeout_ms = group, root, timeout_ms
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.h2, self.w2 = H // 2, W // 2
        self.slot_elems = B * K * self.h2 * self.w2
        self.slot_bytes = 2 * self.slot_elems
        self.step = 0
        self.device = engine.device
        self.comm = torch.cuda.Stream(device=self.device)
        self.done = [None, None]
        self.mode = mode if self.world > 1 else "single"
        self.fallback_reason = None
        self.out = None
        if (self.rank == root or self.world == 1) and materialize:
            self.out = torch.empty((self.world * B, K, H, W), dtype=torch.float32, device=self.device)
        if self.mode.startswith("p2p"):
            try:
                self._setup_p2p()
                ok = 1
            except Exception as e:  # IPC unavailable in this container / topology: every rank must agree to fall back
                ok = 0
                self.fallback_reason = str(e)[:200]
            t = torch.tensor([ok], device=self.device)
            dist.all_reduce(t, op=dist.ReduceOp.MIN, group=group)
            if int(t.item()) == 0:
                self._teardown_p2p()
                self.mode = "nccl"
                self.fallback_reason = self.fallback_reason or "a peer could not map the gather buffer"
        if self.mode == "nccl":
            self.lr = [torch.empty((B, K, self.h2, self.w2), dtype=torch.float16, device=self.device) for _ in range(2)]
            self.gathered = torch.empty((self.world * B, K, self.h2, self.w2), dtype=torch.float16, device=self.device)

    # ---- CUDA IPC setup: one buffer per rank = flag page (+ the two gather slots on root) ----
    def _setup_p2p(self):
        import ctypes as C
        from . import _lib
        lib = self.lib = _lib.load()
        self.base = self.root_base = None
        self.peer_bases = {}
        nbytes = _FLAG_BYTES + (2 * self.world * self.slot_bytes if self.rank == self.root else 0)
        ptr = C.c_void_p()
        handle = C.create_string_buffer(64)
        with torch.cuda.device(self.device):
            _lib.check(lib.lseg_p2p_alloc(nbytes, C.byref(ptr), handle))
        self.base = ptr.value
        handles = [None] * self.world
        dist.all_gather_object(handles, bytes(handle.raw), group=self.group)
        with torch.cuda.device(self.device):
            if self.rank != self.root:
                p = C.c_void_p()
                _lib.check(lib.lseg_p2p_open(handles[self.root], C.byref(p)))
                self.root_base = p.value
                if self.mode == "p2p_copy":
                    self.lr = [torch.empty((self.B, self.K, self.h2, self.w2), dtype=torch.float16, device=self.device)
                               for _ in range(2)]
            else:
                for r in range(self.world):
                    if r == self.root:
                        continue
                    p = C.c_void_p()
                    _lib.check(lib.lseg_p2p_open(handles[r], C.byref(p)))
                    self.peer_bases[r] = p.value

    def _teardown_p2p(self):
        lib = getattr(self, "lib", None)
        if lib is None:
            return
        with torch.cuda.device(self.device):
            torch.cuda.synchronize()
            if getattr(self, "root_base", None):
                lib.lseg_p2p_close(self.root_base)
                self.root_base = None
            for p in getattr(self, "peer_bases", {}).values():
                lib.lseg_p2p_close(p)
            self.peer_bases = {}
            if getattr(self, "base", None):
                lib.lseg_p2p_free(self.base)
                self.base = None

    def close(self):
        if dist.is_initialized() and self.world > 1:
            dist.barrier(group=self.group)  # nobody unmaps while a peer may still write
        self._teardown_p2p()

    def _slot(self, base, parity, r):
        return base + _FLAG_BYTES + (parity * self.world + r) * self.slot_bytes

    # ---- one step ----
    def forward(self, x, text, text_image_stride=0):
        """Enqueue one step. On root returns the fp32 [world*B,K,H,W] logits tensor (complete once `sync()` or an event
        recorded after it has passed; overwritten by the next step); None elsewhere."""
        import ctypes as C
        from . import _lib
        eng = self.engine
        if self.mode == "single":
            return eng.forward(x, text, self.K, text_image_stride, out=self.out)
        self.step += 1
        s, par = self.step, self.step & 1
        cur = torch.cuda.current_stream(self.device)
        if self.done[par] is not None:
            cur.wait_event(self.done[par])  # the buffer / slot of step s-2 is free again
        if self.mode == "nccl":
            eng.forward_lowres(x, text, self.K, text_image_stride, logits_lr=self.lr[par])
            ready = torch.cuda.Event()
            ready.record(cur)
            with torch.cuda.stream(self.comm):
                self.comm.wait_event(ready)
                dist.all_gather_into_tensor(self.gathered, self.lr[par], group=self.group)
                if self.rank == self.root:
                    self._upsample(self.gathered.data_ptr())
                ev = torch.cuda.Event()
                ev.record(self.comm)
            self.done[par] = ev
            return self.out
        lib = self.lib
        cs = C.c_void_p(self.comm.cuda_stream)
        if self.rank != self.root:
            own_consumed = self.base + 8 * _CONSUMED
            if self.mode == "p2p_store":
                if s > 2:
                    _lib.check(lib.lseg_p2p_wait(C.c_void_p(own_consumed), 1, 1, s - 2, self.timeout_ms,
                                                 C.c_void_p(cur.cuda_stream)))
                eng.forward_lowres(x, text, self.K, text_image_stride,
                                   logits_lr=self._slot(self.root_base, par, self.rank))
                _lib.check(lib.lseg_p2p_signal(C.c_void_p(self.root_base + 8 * self.rank), s, C.c_void_p(cur.cuda_stream)))
                return None
            eng.forward_lowres(x, text, self.K, text_image_stride, logits_lr=self.lr[par])
            ready = torch.cuda.Event()
            ready.record(cur)
            with torch.cuda.stream(self.comm):
                self.comm.wait_event(ready)
                if s > 2:
                    _lib.check(lib.lseg_p2p_wait(C.c_void_p(own_consumed), 1, 1, s - 2, self.timeout_ms, cs))
                _lib.check(lib.lseg_p2p_copy(C.c_void_p(self._slot(self.root_base, par, self.rank)),
                                             C.c_void_p(self.lr[par].data_ptr()), self.slot_bytes, cs))
                _lib.check(lib.lseg_p2p_signal(C.c_void_p(self.root_base + 8 * self.rank), s, cs))
                ev = torch.cuda.Event()
                ev.record(self.comm)
            self.done[par] = ev
            return None
        # root
        eng.forward_lowres(x, text, self.K, text_image_stride, logits_lr=self._slot(self.base, par, self.root))
        if self.pipelined:
            if s > 1 and self._expanded < s - 1:
                return self._expand_on(cur, s - 1)
            return self.out if s > 1 else None
        ready = torch.cuda.Event()
        ready.record(cur)
        with torch.cuda.stream(self.comm):
            self.comm.wait_event(ready)
            peers = [r for r in range(self.world) if r != self.root]
            # ready flags of ranks 1.. are contiguous when root == 0; otherwise wait on them one by one
            if self.root == 0:
                _lib.check(lib.lseg_p2p_wait(C.c_void_p(self.base + 8), self.world - 1, 1, s, self.timeout_ms, cs))
            else:
                for r in peers:
                    _lib.check(lib.lseg_p2p_wait(C.c_void_p(self.base + 8 * r), 1, 1, s, self.timeout_ms, cs))
            self._upsample(self._slot(self.base, par, 0))
            for r in peers:
                _lib.check(lib.lseg_p2p_signal(C.c_void_p(self.peer_bases[r] + 8 * _CONSUMED), s, cs))
            ev = torch.cuda.Event()
            ev.record(self.comm)
        self.done[par] = ev
        return self.out

    def _expand_on(self, stream, t):
        """root, pipelined mode: expand the gathered shards of step t on `stream` (the caller's current stream)."""
        import ctypes as C
        from . import _lib
        lib, st = self.lib, C.c_void_p(stream.cuda_stream)
        peers = [r for r in range(self.world) if r != self.root]
        if self.root == 0:
            _lib.check(lib.lseg_p2p_wait(C.c_void_p(self.base + 8), self.world - 1, 1, t, self.timeout_ms, st))
        else:
            for r in peers:
                _lib.check(lib.lseg_p2p_wait(C.c_void_p(self.base + 8 * r), 1, 1, t, self.timeout_ms, st))
        self._upsample(self._slot(self.base, t & 1, 0))
        for r in peers:
            _lib.check(lib.lseg_p2p_signal(C.c_void_p(self.peer_bases[r] + 8 * _CONSUMED), t, st))
        self._expanded = t
        return self.out

    def flush(self):
        """pipelined mode: expand the last step (root) and return the gathered logits; otherwise just sync()."""
        if self.pipelined and self.rank == self.root and self.mode != "single" and self._expanded < self.step:
            self._expand_on(torch.cuda.current_stream(self.device), self.step)
        self.sync()
        return self.out

    def _upsample(self, lr_ptr):
        import ctypes as C
        from . import _lib
        self.lr_ptr = lr_ptr
        if not self.materialize:
            return
        lib = _lib.load()
        # background=True: the shared-memory-free kernel meant to run beside the next step's trunk; the default is the
        # shared-memory kernel (same values bit for bit)
        fn = lib.lseg_upsample2x_nchw_bg if self.background else lib.lseg_upsample2x_nchw
        per = max(1, 65535 // (self.B * self.K))  # images per launch (grid.y limit)
        cs = C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

        def expand(img0, n_img):
            off = img0 * self.K
            _lib.check(fn(C.c_void_p(lr_ptr + 2 * off * self.h2 * self.w2),
                          C.c_void_p(self.out.data_ptr() + 4 * off * self.H * self.W), n_img * self.K, self.h2, self.w2, cs))

        for _ in range(self.repeat):
            if self.root_batch < self.B and self.root == 0:  # own (short) shard, then the peers' slots
                expand(0, self.root_batch)
                first = 1
            else:
                first = 0
            for r0 in range(first, self.world, per):
                expand(r0 * self.B, min(per, self.world - r0) * self.B)

    def sync(self):
        """Make the current stream wait for everything this object has enqueued on its side stream."""
        torch.cuda.current_stream(self.device).wait_stream(self.comm)
