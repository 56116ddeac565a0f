"""The fused multi-GPU traversal step (bvhgpu_traverse_sharded_dev_*, traverse.cu §"exchange over peer memory") restated and driven
from one process (test infrastructure).

Layout restatement (numpy, no GPU): rays and tiles before every source rank, the count width of a tile, the bytes of one staging
half (the counts of tile g at 8192 g in the tile's width, the table entry `offset | width << 56` at table_off + 8 g) and the mailbox
words a step leaves.

VirtualShards: W "ranks" in one process on one GPU.  The shard struct takes raw device pointers, so every rank's buffers can live on
the same device: each rank gets its own Context (own stream, own replica of the tree), its own peer-allocated staging, hit buffer,
mailbox and offsets (each followed by a canary guard), and every step is enqueued by one host thread per rank (ctypes releases the
GIL, so no rank's enqueue waits on another's).  Two ranks never share a context: one stream would run them one after the other, and
the first would wait out the exchange time-out for a peer queued behind it."""
import ctypes as C
import threading

import numpy as np

from oracle import oracle as O

TILE = 2048                 # SCAN_TILE: rays per tile, counted from the first ray of each source rank
TILE_BYTES = 4 * TILE       # bytes reserved for the counts of one tile (room for the 4-byte width)
MAX_PEERS = 8
MB_TOT, MB_DONE, MB_TRACE, MB_TRACE_LEN = 0, 64, 128, 1024       # mailbox word offsets (u64)
GUARD = 256                 # canary bytes behind every buffer of the harness
CANARY = 0xA5


# ---- layout restatement -----------------------------------------------------------------------------------------------------
def rays_before(sizes) -> np.ndarray:
    return np.concatenate([[0], np.cumsum(np.asarray(sizes, dtype=np.int64))])


def tiles_before(sizes) -> np.ndarray:
    return np.concatenate([[0], np.cumsum([(int(n) + TILE - 1) // TILE for n in sizes])]).astype(np.int64)


def width(largest: int) -> int:
    """Bytes per staged count of a tile whose largest count is `largest`."""
    return 1 if largest <= 0xFF else (2 if largest <= 0xFFFF else 4)


def layout_bytes(sizes) -> int:
    """Bytes of one staging half the layout uses: the count slots of every tile, then the tile table."""
    nt = int(tiles_before(sizes)[-1])
    return TILE_BYTES * nt + 8 * nt


def stage_bytes(nrays_global: int) -> int:
    """BVHGPU_SHARD_STAGE_BYTES restated (bvh_b200.h)."""
    return (8200 * (nrays_global // 2048 + 2 * MAX_PEERS) + 255) & ~255


def tiles(sizes, counts):
    """One tuple per global tile g: (g, source rank, first global ray, rays in the tile, largest count, width, exclusive hit offset of
    the tile inside its source's list).  counts: the per-ray hit counts of the whole batch in global ray order."""
    counts = np.asarray(counts, dtype=np.int64)
    rb, tb = rays_before(sizes), tiles_before(sizes)
    out = []
    for s, n in enumerate(sizes):
        off = 0
        for t in range((int(n) + TILE - 1) // TILE):
            lo = int(rb[s]) + t * TILE
            c = counts[lo: min(lo + TILE, int(rb[s + 1]))]
            m = int(c.max()) if len(c) else 0
            out.append((int(tb[s]) + t, s, lo, len(c), m, width(m), off))
            off += int(c.sum())
    return out


def staging_image(sizes, counts):
    """(image, written): the bytes of one staging half after a step over `counts`, and a mask of the bytes that step writes (a count
    slot keeps what an earlier, wider step left behind its own width)."""
    counts = np.asarray(counts, dtype=np.int64)
    nt = int(tiles_before(sizes)[-1])
    table_off = TILE_BYTES * nt
    img = np.zeros(table_off + 8 * nt, dtype=np.uint8)
    written = np.zeros(len(img), dtype=bool)
    for g, _s, lo, n, _m, w, off in tiles(sizes, counts):
        c = np.zeros(TILE, dtype=np.uint64)
        c[:n] = counts[lo: lo + n]
        enc = c.astype({1: "<u1", 2: "<u2", 4: "<u4"}[w]).view(np.uint8)
        img[TILE_BYTES * g: TILE_BYTES * g + TILE * w] = enc
        written[TILE_BYTES * g: TILE_BYTES * g + TILE * w] = True
        e = np.array([off | (w << 56)], dtype="<u8").view(np.uint8)
        img[table_off + 8 * g: table_off + 8 * g + 8] = e
        written[table_off + 8 * g: table_off + 8 * g + 8] = True
    return img, written


def mailbox_words(seq: int, totals) -> dict:
    """{u64 word: value} that a step with sequence number `seq` leaves in EVERY rank's mailbox (trace: the seq word only)."""
    par = seq & 1
    words = {}
    for src, tot in enumerate(totals):
        words[MB_TOT + (par * MAX_PEERS + src) * 4] = seq
        words[MB_TOT + (par * MAX_PEERS + src) * 4 + 1] = int(tot)
        words[MB_DONE + par * MAX_PEERS + src] = seq
    words[MB_TRACE + (seq % MB_TRACE_LEN) * 4] = seq
    return words


def global_csr(offsets, hits):
    """The oracle's CSR as (u32 offsets, u32 hits) as a rank holds it (offsets at or past 2^32 read 0xFFFFFFFF)."""
    off = np.minimum(np.asarray(offsets, dtype=np.uint64), np.uint64(0xFFFFFFFF)).astype(np.uint32)
    return off, np.asarray(hits, dtype=np.uint32)


def od_layout(rays: np.ndarray) -> np.ndarray:
    """BVHGPU_RAYS_OD: origin and direction, 6 scalars per ray."""
    od = np.empty((len(rays), 6), dtype=rays["origin"].dtype)
    od[:, :3], od[:, 3:] = rays["origin"], rays["direction"]
    return od


def oracle_csr(shapes, rays, mode: int, prec: str):
    """O.traverse of the concatenated batch: MODE_RECURSIVE for TRAVERSE_BVH (0), MODE_FLAT on the flattened tree for TRAVERSE_FLAT."""
    nodes = O.build(shapes, prec).nodes
    if mode == 0:
        return O.traverse(nodes, shapes, rays, O.MODE_RECURSIVE, prec, threads=8)
    return O.traverse(O.flatten(nodes, prec), shapes, rays, O.MODE_FLAT, prec, threads=8)


# ---- inputs shared by the in-process tests and the multi-process check ------------------------------------------------------
def uneven(ng, w):
    """ng rays over w ranks, uneven: rank r gives (r % 3) + 1 rays to rank r + 1, so shards start at offsets that are not multiples
    of 4."""
    sizes = [ng // w + (1 if r < ng % w else 0) for r in range(w)]
    for r in range(0, w - 1, 2):
        k = min(r % 3 + 1, sizes[r] - 1)
        sizes[r] -= k
        sizes[r + 1] += k
    return sizes


def miss_rays(shapes, n, prec, seed):
    """Rays that start beyond the scene's upper corner and point away from it: no box is hit."""
    rng = np.random.default_rng(seed)
    mn, mx = shapes["min"].astype(np.float64), shapes["max"].astype(np.float64)
    lo, hi = mn.min(axis=0), mx.max(axis=0)
    org = hi + (hi - lo) * rng.uniform(0.5, 1.0, (n, 3))
    return O.ray_new(org, rng.uniform(0.1, 1.0, (n, 3)), prec)


def pile(n, prec="f32", seed=0):
    """n boxes that all contain the origin."""
    rng = np.random.default_rng(seed + n)
    half = rng.uniform(1.0, 2.0, (n, 3))
    return O.make_aabbs(-half * rng.uniform(0.5, 1.0, (n, 3)), half, prec)


def pile_rays(ng, through, prec="f32", seed=0):
    """ng rays from a sphere of radius 20..40: those listed in `through` point at the origin (they hit every box of a pile), the
    others point away (they hit nothing)."""
    rng = np.random.default_rng(seed)
    org = rng.normal(size=(ng, 3))
    org *= rng.uniform(20, 40, (ng, 1)) / np.linalg.norm(org, axis=1, keepdims=True)
    dirs = org.copy()
    dirs[through] = -org[through]
    return O.ray_new(org, dirs, prec)


def line_scene(k=600, prec="f32"):
    """k unit boxes along x, 10 apart: a ray up the z axis through a box's column hits that box only."""
    x = 10.0 * np.arange(k)
    mn = np.stack([x, np.zeros(k), np.zeros(k)], axis=1)
    return O.make_aabbs(mn, mn + 1.0, prec)


def line_rays(sizes, seed=0, prec="f32"):
    """Per rank, per 256-ray emit block b: (b + rank + 1) % 8 rays that hit one box each (a hit piece of 0 to 7 words), every 11th block
    9 to 40 of them (quads with a head and a tail), at random places in the block; the other rays miss."""
    rng = np.random.default_rng(seed)
    ng = sum(sizes)
    hit = np.zeros(ng, dtype=bool)
    rb = rays_before(sizes)
    for r, n in enumerate(sizes):
        for b in range((n + 255) // 256):
            m = min(256, n - 256 * b)
            k = (b + r + 1) % 8 if b % 11 != 10 else int(rng.integers(9, 41))
            hit[rb[r] + 256 * b + rng.choice(m, min(k, m), replace=False)] = True
    box = rng.integers(0, 600, ng)
    org = np.stack([10.0 * box + 0.5, np.where(hit, 0.5, 5.0), np.full(ng, -5.0)], axis=1)
    dirs = np.tile([0.0, 0.0, 1.0], (ng, 1))
    return O.ray_new(org, dirs, prec)


# ---- in-process harness ---------------------------------------------------------------------------------------------------------
class VirtualShards:
    """W ranks of the fused step on one GPU.  sizes: rays of every rank's shard (fixed for the harness's life); cap: capacity of the
    global hit buffers; layout: capi.RAYS_FULL / RAYS_OD; mode: capi.TRAVERSE_BVH / TRAVERSE_FLAT."""

    def __init__(self, shapes, sizes, cap: int, prec: str = "f32", layout: int = 0, mode: int = 0):
        import torch

        from bvh_b200 import api, capi

        self.torch, self.api, self.capi = torch, api, capi
        self.L = capi.lib()
        self.sizes = [int(n) for n in sizes]
        self.W, self.NG, self.cap = len(self.sizes), sum(self.sizes), int(cap)
        assert 1 <= self.W <= MAX_PEERS
        self.prec, self.layout, self.mode = prec, layout, mode
        self.dev = torch.device("cuda", 0)
        self.half = capi.shard_stage_bytes(self.NG)
        self.nbytes = {"stage": 2 * self.half, "hits": 4 * self.cap, "box": capi.MAILBOX_BYTES, "offsets": 4 * (self.NG + 1)}
        self.ctxs, self.streams, self.bvhs, self.bufs, self.shards = [], [], [], [], []
        self.seq = 0
        try:
            for r in range(self.W):
                ctx = api.Context(0)
                self.ctxs.append(ctx)
                st = torch.cuda.Stream(self.dev)
                self.streams.append(st)
                ctx.set_stream(st.cuda_stream)
                self.bvhs.append(api.Bvh.build(shapes, prec=prec, ctx=ctx))
                bufs = {}
                for name, nb in self.nbytes.items():
                    p, h = C.c_void_p(), (C.c_ubyte * capi.IPC_HANDLE_BYTES)()
                    capi.check(self.L.bvhgpu_peer_alloc(ctx._h, nb + GUARD, C.byref(p), h))
                    bufs[name] = p
                    g = np.full(GUARD, CANARY, dtype=np.uint8)
                    capi.check(self.L.bvhgpu_memcpy_h2d_async(ctx._h, C.c_void_p(p.value + nb), g.ctypes.data_as(C.c_void_p), GUARD))
                ctx.synchronize()
                self.bufs.append(bufs)
            for r in range(self.W):
                s = capi.Shard()
                s.rank, s.world, s.cap, s.seq, s.ray_layout = r, self.W, self.cap, 0, int(layout)
                s.offsets = self.bufs[r]["offsets"].value
                for d in range(self.W):
                    s.shard_rays[d] = self.sizes[d]
                    s.peer_counts[d] = self.bufs[d]["stage"].value
                    s.peer_hits[d] = self.bufs[d]["hits"].value
                    s.peer_mailbox[d] = self.bufs[d]["box"].value
                self.shards.append(s)
            self.fn = getattr(self.L, f"bvhgpu_traverse_sharded_dev_{self.bvhs[0]._d['suffix']}")
        except BaseException:
            self.close()
            raise

    # rays --------------------------------------------------------------------------------------------------------------------------
    def upload(self, rays: np.ndarray):
        """The batch (global ray order) cut into the ranks' shards, on the device in the harness's layout: one tensor per rank."""
        assert len(rays) == self.NG
        rb = rays_before(self.sizes)
        out = []
        for r in range(self.W):
            part = rays[rb[r]: rb[r + 1]]
            host = od_layout(part) if self.layout == self.capi.RAYS_OD else part
            out.append(self.torch.from_numpy(np.ascontiguousarray(host).view(np.uint8).reshape(-1)).to(self.dev))
        self.torch.cuda.synchronize(self.dev)
        return out

    def warm_up(self, d_rays):
        """A plain traverse_dev of each rank's shard on its own context: the traversal records, the top records and the slot budget
        are built here, not inside the first sharded step.  (traverse_dev takes full rays; the OD layout warms up through the
        od entry point.)"""
        for r in range(self.W):
            n = self.sizes[r]
            off = self.torch.empty(n + 1, dtype=self.torch.int32, device=self.dev)
            hits = self.torch.empty(4 * n + 16, dtype=self.torch.int32, device=self.dev)
            fn = "traverse_dev" if self.layout == self.capi.RAYS_FULL else "traverse_od_dev"
            f = getattr(self.L, f"bvhgpu_{fn}_{self.bvhs[r]._d['suffix']}")
            self.capi.check(f(self.bvhs[r]._h, self.mode, C.c_void_p(d_rays[r].data_ptr()), n, C.c_void_p(off.data_ptr()),
                              C.c_void_p(hits.data_ptr()), hits.numel(), None))
            self.ctxs[r].synchronize()

    # one step ----------------------------------------------------------------------------------------------------------------------
    def step(self, d_rays, straggler: int | None = None, sleep_cycles: int = 100_000_000):
        """Enqueue one step on every rank, each from its own host thread.  straggler: a rank whose stream first sleeps for
        `sleep_cycles` (a bounded torch.cuda._sleep, about 0.1 s), so that its peers reach the hand-shakes long before it does."""
        self.seq += 1
        status = [None] * self.W

        def enqueue(r):
            s = self.shards[r]
            s.seq = self.seq
            if r == straggler:
                with self.torch.cuda.stream(self.streams[r]):
                    self.torch.cuda._sleep(sleep_cycles)
            status[r] = self.fn(self.bvhs[r]._h, self.mode, C.c_void_p(d_rays[r].data_ptr()), self.sizes[r], C.byref(s))

        threads = [threading.Thread(target=enqueue, args=(r,)) for r in range(self.W)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        for r, st in enumerate(status):
            if st != self.capi.OK:
                self.synchronize()
                self.capi.check(st)

    def synchronize(self):
        """Wait for every rank; a time-out of the exchange is raised once, as bvhgpu_synchronize reports it (never retried)."""
        err = None
        for ctx in self.ctxs:
            try:
                ctx.synchronize()
            except self.capi.BvhGpuError as e:
                err = err or e
        if err is not None:
            raise err

    # read-back ---------------------------------------------------------------------------------------------------------------------
    def _read(self, r, name, nbytes, offset=0):
        out = np.empty(nbytes, dtype=np.uint8)
        if nbytes:
            self.capi.check(self.L.bvhgpu_memcpy_d2h(self.ctxs[r]._h, out.ctypes.data_as(C.c_void_p),
                                                     C.c_void_p(self.bufs[r][name].value + offset), nbytes))
        return out

    def offsets(self, r) -> np.ndarray:
        return self._read(r, "offsets", 4 * (self.NG + 1)).view(np.uint32)

    def hits(self, r, n=None) -> np.ndarray:
        return self._read(r, "hits", 4 * (self.cap if n is None else n)).view(np.uint32)

    def staging(self, r, seq=None) -> np.ndarray:
        """The staging half of step `seq` (default: the last step) in rank r's buffer."""
        par = (self.seq if seq is None else seq) & 1
        return self._read(r, "stage", self.half, par * self.half)

    def mailbox(self, r) -> np.ndarray:
        return self._read(r, "box", self.capi.MAILBOX_BYTES).view(np.uint64)

    def guards_intact(self) -> bool:
        return all(np.all(self._read(r, name, GUARD, nb) == CANARY) for r in range(self.W) for name, nb in self.nbytes.items())

    def fetch(self, r):
        """ShardedTraversal.fetch on rank r: the global CSR, or BvhGpuError(ERR_CAPACITY) when the u32 offsets overflowed or the
        hits do not fit `cap`."""
        off = self.offsets(r)
        total = int(off[self.NG])
        if total == 0xFFFFFFFF:
            raise self.capi.BvhGpuError(self.capi.ERR_CAPACITY, "sharded traversal: the hit total overflows the u32 CSR offsets")
        if total > self.cap:
            raise self.capi.BvhGpuError(self.capi.ERR_CAPACITY, f"sharded traversal: {total} hits do not fit cap {self.cap}")
        return off, self.hits(r, total)

    def trace(self, r) -> dict:
        box = self.mailbox(r)
        tr = box[MB_TRACE: MB_TRACE + 4 * MB_TRACE_LEN].reshape(-1, 4)
        return {int(t[0]): i for i, t in enumerate(tr) if t[0] != 0}

    def close(self):
        try:
            self.synchronize()
        except Exception:
            pass
        for r, bufs in enumerate(self.bufs):
            for p in bufs.values():
                self.L.bvhgpu_peer_free(self.ctxs[r]._h, p)
        self.bufs = []
        for b in self.bvhs:
            b.free()
        self.bvhs = []
        for ctx in self.ctxs:
            ctx.close()
        self.ctxs = []
