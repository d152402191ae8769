"""Multi-GPU host logic: frames (monitors) shard across ranks, no data-path collective.

crt_modulate / crt_demodulate of different `struct CRT` instances never exchange data, so the
N-GPU path is one process per GPU (torchrun), each advancing its own contiguous slice of the batch;
torch.distributed is used only for the barrier, the max-over-ranks timing and -- optionally -- to
all_gather the decoded frames when a caller wants every rank to hold the whole batch (the exchange
BASELINE.json's north_star mentions; it is NVLink-bound, see DESIGN.md section 6).
"""
import os


def rank_info():
    """(rank, local_rank, world_size) from the torchrun environment; (0, 0, 1) standalone."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")),
            int(os.environ.get("WORLD_SIZE", "1")))


def shard_range(n_items, rank, world):
    """Contiguous [lo, hi) of rank's items; sizes differ by at most one, earlier ranks larger."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def max_over_ranks(values, device=None, group=None):
    """Element-wise max of a list of floats over all ranks (timings are max-over-ranks)."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return list(values)
    t = torch.tensor(list(values), dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX, group=group)
    return [float(x) for x in t]


def allgather_frames(local, group=None):
    """all_gather equally-shaped per-rank frame tensors -> (world * n_local, ...) on every rank."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return local
    world = dist.get_world_size(group)
    out = torch.empty((world,) + tuple(local.shape), dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out.view(-1), local.contiguous().view(-1), group=group)
    return out.view((world * local.shape[0],) + tuple(local.shape[1:]))


# ---------------------------------------------------------------------------------------------
# One image over several GPUs: scanline blocks
# ---------------------------------------------------------------------------------------------
# The fields of ONE image are sequentially dependent through the blend (crt_core.c:584-608), so a single
# image cannot be spread over ranks by field.  Its decoded scanlines can: after the sync pre-pass every
# line is independent (crt_core.c:409-664), and line k of a field only touches output rows
#     beg = k * (outh + v_fac) / CRT_LINES + field  ..  end = (k + 1) * (outh + v_fac) / CRT_LINES + field
# (crt_core.c:428-432, rows beg .. end - scanlines - 1 are written).  Every rank runs the SAME calls --
# modulate, noise, sync search are replicated, they are a small part of the work -- with the line pass
# restricted to its block (crtx_set_option "line_lo"/"line_hi") and keeps the accumulation of its own rows
# across the fields; one all_gather of row blocks at the end gives every rank the whole image.
#
# The one coupling between blocks: in an odd field every line is shifted down by field * (ratio / 2) rows
# (crt_core.c:400-407), so the last line of a block may write (duplicate into) the first rows of the
# NEXT block -- rows the next even field of that block blends with.  `exchange_spill_rows` hands those
# few rows to the neighbour after each field.

def line_block(rank, world, lines):
    """Decoded scanlines [lo, hi) of `rank` (contiguous, sizes differ by at most one)."""
    return shard_range(lines, rank, world)


def row_span(outh, v_fac, lines):
    """outh + v_fac as the reference computes it, in 32-bit unsigned arithmetic (v_fac is unsigned, crt_core.c:428):
    a "negative" v_fac shrinks the span.  Raises ValueError for a span at which (k + 1) * span wraps 32 bits for some
    line: lines far apart then share rows, and no partition into blocks of consecutive lines keeps their order."""
    span = (outh + v_fac) & 0xFFFFFFFF
    if span > 0xFFFFFFFF // lines:
        raise ValueError("outh + v_fac = %d rows: the reference's row mapping wraps 32 bits, lines far apart share rows" % span)
    return span


def block_rows(lo, hi, outh, lines, v_fac=0):
    """Output rows [r0, r1) owned by the rank decoding lines [lo, hi): the rows its lines start on in an
    even field (crt_core.c:428), clipped to the image."""
    span = row_span(outh, v_fac, lines)
    return min(outh, lo * span // lines), min(outh, hi * span // lines)


class ImageSharder:
    """Row ownership and the exchanges of the scanline-block partition of one image.

    image: this rank's (outh, outw, bpp) uint8 tensor (any device the process group supports).

    Per field:  fetch_halo_rows()  ->  the decode of this rank's lines  ->  exchange_spill_rows(written_end).
    In an odd field every line is shifted down by ratio / 2 rows (crt_core.c:400-407), so the last line of a block
    reaches into the first rows of the NEXT block: it may only duplicate into them (a taller line) or -- when the line
    is no taller than the shift -- put its COMPUTED row there, which the blend mixes with what that row held
    (crt_core.c:584-608).  That content is the next rank's, so the next rank lends it first (the halo) and gets the
    result back (the spill)."""

    def __init__(self, image, lines, rank=None, world=None, v_fac=0, group=None):
        import torch.distributed as dist
        self.group = group
        on = dist.is_available() and dist.is_initialized()
        self.world = world if world is not None else (dist.get_world_size(group) if on else 1)
        self.rank = rank if rank is not None else (dist.get_rank(group) if on else 0)
        self.image, self.lines, self.v_fac = image, lines, v_fac
        self.outh = image.shape[0]
        span = row_span(self.outh, v_fac, lines)
        if self.world > 1 and span < lines:
            # several decoded lines share an output row and the reference applies them in line order
            # (crt_core.c:409-664 is a sequential loop): lines of two ranks would have to take turns on one row
            raise ValueError("scanline-block sharding needs at least one output row per decoded line: outh + v_fac = %d < %d lines"
                             % (span, lines))
        self.lo, self.hi = line_block(self.rank, self.world, lines)
        self.blocks = [block_rows(*line_block(r, self.world, lines), self.outh, lines, v_fac)
                       for r in range(self.world)]
        self.r0, self.r1 = self.blocks[self.rank]
        if self.world > 1 and min(b - a for a, b in self.blocks) < self.max_spill():
            raise ValueError("scanline-block sharding: %d ranks leave a block with fewer than %d rows (the odd-field shift), "
                             "use fewer ranks for a %d-row image" % (self.world, self.max_spill(), self.outh))

    def apply(self, batch):
        """Restrict a capi.Batch's line pass to this rank's block."""
        batch.set_option("line_lo", self.lo)
        batch.set_option("line_hi", self.hi)

    def max_spill(self):
        """Most rows a block can reach into its successor: the odd-field shift ratio / 2 of crt_core.c:404-407 (the
        ratio is taken from outh alone there; v_fac only stretches beg / end, crt_core.c:428-429)."""
        ratio = (((self.outh << 16) // self.lines) + 32768) >> 16
        return max(1, ratio // 2)

    def _halo_count(self, r):
        """rows rank r borrows from rank r + 1: the first max_spill() rows of that block"""
        if r + 1 >= self.world or self.blocks[r + 1][0] != self.blocks[r][1]:
            return 0
        a, b = self.blocks[r + 1]
        return max(0, min(self.max_spill(), b - a))

    def fetch_halo_rows(self):
        """Before a field: the first max_spill() rows of the next rank's block, as that rank holds them now, into this
        rank's image -- what this rank's last line will blend with if its computed row lands there.  One small
        all_gather.  (Cheap enough to do before every field; only odd fields of blended images need it.)"""
        import torch
        import torch.distributed as dist
        if self.world == 1:
            return
        cap = self.max_spill()
        mine = torch.zeros((cap,) + tuple(self.image.shape[1:]), dtype=self.image.dtype, device=self.image.device)
        n_mine = min(cap, self.r1 - self.r0)
        if n_mine:
            mine[:n_mine].copy_(self.image[self.r0:self.r0 + n_mine])
        rows = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(rows, mine, group=self.group)
        cnt = self._halo_count(self.rank)
        if cnt:
            self.image[self.r1:self.r1 + cnt].copy_(rows[self.rank + 1][:cnt])

    def exchange_spill_rows(self, written_end):
        """After a field.  written_end: one past the last output row this rank's LAST line wrote in this
        field (`end - scanlines` of line hi - 1 from the sync table, or anything <= r1 if it was skipped).
        Rows [r1, written_end) belong to the next rank, which takes them into its image.  Two small
        all_gathers (the rows, and how many of them count)."""
        import torch
        import torch.distributed as dist
        if self.world == 1:
            return
        cap = self.max_spill()
        cnt = max(0, min(int(written_end), self.outh, self.r1 + cap) - self.r1) if self.rank + 1 < self.world else 0
        mine = torch.zeros((cap,) + tuple(self.image.shape[1:]), dtype=self.image.dtype, device=self.image.device)
        if cnt:
            mine[:cnt].copy_(self.image[self.r1:self.r1 + cnt])
        rows = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(rows, mine, group=self.group)
        n_mine = torch.tensor([cnt], dtype=torch.int64, device=self.image.device)
        counts = [torch.empty_like(n_mine) for _ in range(self.world)]
        dist.all_gather(counts, n_mine, group=self.group)
        if self.rank > 0 and self.blocks[self.rank - 1][1] == self.r0:
            got = int(counts[self.rank - 1].item())
            if got:
                self.image[self.r0:self.r0 + got].copy_(rows[self.rank - 1][:got])

    def gather(self):
        """Every rank's own rows -> the complete image on every rank (blocks padded to equal height)."""
        import torch
        import torch.distributed as dist
        if self.world == 1:
            return self.image
        tall = max(b - a for a, b in self.blocks)
        mine = torch.zeros((tall,) + tuple(self.image.shape[1:]), dtype=self.image.dtype, device=self.image.device)
        mine[:self.r1 - self.r0].copy_(self.image[self.r0:self.r1])
        parts = [torch.empty_like(mine) for _ in range(self.world)]
        dist.all_gather(parts, mine, group=self.group)
        full = self.image.clone()
        for r, (a, b) in enumerate(self.blocks):
            full[a:b].copy_(parts[r][:b - a])
        return full
