"""Multi-GPU partitioning of the frame-analysis path (host logic only; one process per GPU).

Frame shards (the reference's frame-parallel mode, -F): each rank analyses its own frame against its own nearest
reference frames: no data-path collective inside a frame.  The single exchange step is the broadcast of the newest
reconstructed reference plane from the rank that owns (reconstructed) it -- the producer side of m_reconRowFlag
(/root/reference/source/encoder/framefilter.cpp:664) -- once per step."""


def frame_of(step, rank, world, first=0):
    """Display index of the frame rank `rank` analyses in step `step` (frames are dealt round-robin)."""
    return first + step * world + rank


def ref_owner(step, world):
    """Rank that holds the newest reconstructed reference plane for step `step`."""
    return step % world


def exchange_ref(dist, plane_tensor, step, world, recv=None):
    """Broadcast the newest reference plane (whole padded allocation, margins included) from its owner.
    `dist` is torch.distributed (NCCL on GPUs, gloo in the CPU tests).  With `recv`, the non-owners receive into that
    tensor (an incoming-reference plane the caller swaps in when it wants to) instead of overwriting `plane_tensor`."""
    if world <= 1:
        return plane_tensor
    owner = ref_owner(step, world)
    t = plane_tensor if (recv is None or dist.get_rank() == owner) else recv
    dist.broadcast(t, src=owner)
    return t


# ---- CTU-row shards inside one frame (BASELINE configs[4]: WPP CTU rows sharded per GPU) -----------------------
# A frame's CTU rows are dealt to the ranks; each rank analyses its rows with x265cu_analyser_run_rows() and owns
# their reconstructed pixels.  The one exchange is the broadcast of every owner's reconstructed rows (the
# producer side of m_reconRowFlag, /root/reference/source/encoder/framefilter.cpp:664; the consumer waits on
# refpic->m_reconRowFlag[row + m_refLagRows], frameencoder.cpp:850-868).  Sharding changes placement only:
# every row's arithmetic is the same slice of the same launch lists, so results do not depend on N.

def row_blocks(nrows, rank, world, mode="block"):
    """CTU-row ranges [(r0, r1), ...] owned by `rank`.
    "block": one contiguous chunk per rank (sizes differ by at most one row) -- one launch set per frame;
    "cyclic": row r belongs to rank r % world -- the order a WPP wavefront releases rows in."""
    if mode == "block":
        base, extra = divmod(nrows, world)
        r0 = rank * base + min(rank, extra)
        r1 = r0 + base + (1 if rank < extra else 0)
        return [(r0, r1)] if r1 > r0 else []
    if mode == "cyclic":
        return [(r, r + 1) for r in range(rank, nrows, world)]
    raise ValueError("unknown row shard mode %r" % mode)


def row_owner(row, nrows, world, mode="block"):
    for g in range(world):
        for r0, r1 in row_blocks(nrows, g, world, mode):
            if r0 <= row < r1:
                return g
    raise ValueError("row %d outside the frame" % row)


def band_slice(r0, r1, height, stride, margin_y, es=1, ctu=64):
    """Byte range, inside a margin-extended plane allocation, of the picture rows of CTU rows [r0, r1)
    (whole stride rows: one contiguous band)."""
    y0, y1 = r0 * ctu, min(height, r1 * ctu)
    return (margin_y + y0) * stride * es, (margin_y + y1) * stride * es


def exchange_rows(dist, plane_tensor, nrows, world, height, stride, margin_y, es=1, mode="block"):
    """Every rank broadcasts the bands of `plane_tensor` (flat uint8 view of a whole plane allocation) it owns;
    afterwards every rank holds the complete plane.  Broadcast only, as in the single-plane exchange."""
    if world <= 1:
        return plane_tensor
    works = []
    for g in range(world):
        for r0, r1 in row_blocks(nrows, g, world, mode):
            b0, b1 = band_slice(r0, r1, height, stride, margin_y, es)
            works.append(dist.broadcast(plane_tensor[b0:b1], src=g, async_op=True))
    for w in works:
        w.wait()
    return plane_tensor


# ---- in-loop filtering of row shards (include/x265_b200.h, x265cu_deblock_rows / _sao_stats_rows / _sao_apply_rows) ----
# A band's deblocking reads and writes pre-deblock luma rows [Y0 - 4, Y1 + 4) and chroma rows [C0 - 4, C1 + 4), so before it
# each rank needs only the 4 luma and 4 chroma rows on either side of its bands from the neighbours that own them; the
# statistics and the apply then read only rows the rank's own deblocking wrote.  Per frame a row shard runs: run_rows,
# exchange_halos of the reconstruction, deblock_rows (recon -> per-rank deblocked scratch), sao_stats_rows, the host's SAO
# decision, sao_apply_rows (scratch -> the resident reference band), exchange_rows of the final bands, ref_updated.

def filter_halo(r0, r1, ctu, height):
    """((y0, y1), (c0, c1)): the luma and 4:2:0 chroma rows x265cu_deblock_rows reads (and writes) for CTU rows [r0, r1)."""
    Y0, Y1 = r0 * ctu, min(height, r1 * ctu)
    return (max(0, Y0 - 4), min(height, Y1 + 4)), (max(0, Y0 // 2 - 4), min(height // 2, Y1 // 2 + 4))


def halo_sends(nrows, world, height, ctu, mode="block"):
    """[(src_rank, (y0, y1), (c0, c1)), ...]: the pre-deblock luma / chroma rows each owner broadcasts so that every rank
    holds the halos of its bands.  At every boundary between CTU rows of different owners, each side sends the 4 luma and 4
    chroma rows next to it (a CTU row is at least 8 luma rows high, so they are the owner's own rows)."""
    out = []
    for r in range(1, nrows):
        above, below = row_owner(r - 1, nrows, world, mode), row_owner(r, nrows, world, mode)
        if above == below:
            continue
        y, c = r * ctu, r * ctu // 2
        out.append((above, (y - 4, y), (c - 4, c)))
        out.append((below, (y, min(height, y + 4)), (c, min(height // 2, c + 4))))
    return out


def exchange_halos(dist, luma, chroma, nrows, world, height, ctu, stride, cstride=0, margin_y=0, cmargin_y=0, es=1,
                   mode="block"):
    """Broadcast-only exchange of the pre-deblock halo rows (halo_sends) between the ranks of a row shard.  `luma`: flat
    uint8 view of the whole luma plane allocation (row stride `stride` pixels, picture row 0 at allocation row `margin_y`);
    `chroma`: () or the (cb, cr) allocations likewise with `cstride` / `cmargin_y`; `es` bytes per pixel.  Returns the
    number of bytes broadcast."""
    if world <= 1:
        return 0
    works, nbytes = [], 0
    for src, (y0, y1), (c0, c1) in halo_sends(nrows, world, height, ctu, mode):
        parts = [(luma, y0, y1, stride, margin_y)] + [(p, c0, c1, cstride, cmargin_y) for p in chroma]
        for t, a, b, st, my in parts:
            b0, b1 = (my + a) * st * es, (my + b) * st * es
            works.append(dist.broadcast(t[b0:b1], src=src, async_op=True))
            nbytes += b1 - b0
    for w in works:
        w.wait()
    return nbytes
