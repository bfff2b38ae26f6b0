"""Host emulation of the depth-order key emit in csrc/binning.cu (emit_keys_kernel): the runs of a warp's 32 depth ranks are
adjacent in the entry sequence, the runs of small AABBs are laid end to end and written 32 consecutive entries per step,
each entry found by an owner search over the exclusive prefix and a bit extraction from the owner's touch mask.  Checks
the index arithmetic, the truncation at the buffer end and the tail padding of the capped form against a per-lane loop."""
import numpy as np

COOP_AREA = 32
TILES_X = 40
SENTINEL = 0xFFFF


def nth_set_bit(m, k):
    pos = 0
    for w in (16, 8, 4, 2, 1):
        c = bin(m & ((1 << w) - 1)).count("1")
        if k >= c:
            k -= c
            m >>= w
            pos += w
    return pos


def emulated(starts, counts, masks, bbs, payloads, big_tiles, end, total, keys, vals):
    """One warp, mirroring the kernel's loop structure.  big_tiles(lane) -> the tiles an AABB above COOP_AREA reaches."""
    n = np.where(starts >= end, 0, counts)
    bwid = bbs[:, 2] - bbs[:, 0]
    area = bwid * (bbs[:, 3] - bbs[:, 1])
    mine = np.array([bin(int(masks[l])).count("1") if n[l] > 0 and area[l] <= COOP_AREA else 0 for l in range(32)])
    pre = np.concatenate([[0], np.cumsum(mine)[:-1]])
    flat = int(mine.sum())
    delta = starts - pre
    tbase = bbs[:, 1] * TILES_X + bbs[:, 0]
    for base in range(0, flat, 32):
        for lane in range(32):
            f = base + lane
            o = 0
            for step in (16, 8, 4, 2, 1):
                cand = o + step
                if pre[cand] <= f:
                    o = cand
            pos = f + delta[o]
            if f < flat and pos < end:
                k = f - pre[o]
                bit = nth_set_bit(int(masks[o]), k)
                w = int(bwid[o])
                r = int((np.float32(bit) + np.float32(0.5)) / np.float32(w))
                assert r == bit // w and (int(masks[o]) >> bit) & 1
                keys[pos] = tbase[o] + r * TILES_X + (bit - r * w)
                vals[pos] = payloads[o]
    for src in range(32):
        if n[src] > 0 and area[src] > COOP_AREA:
            pos = starts[src]
            for tile in big_tiles(src):
                if pos < end:
                    keys[pos] = tile
                    vals[pos] = payloads[src]
                pos += 1
    if total is not None:
        keys[min(total, end):end] = SENTINEL
        vals[min(total, end):end] = 0


def per_lane(starts, masks, bbs, payloads, big_tiles, end, total, keys, vals):
    """The row-order form: each lane walks its own AABB."""
    for lane in range(32):
        x0, y0, x1, y1 = (int(v) for v in bbs[lane])
        w, area = x1 - x0, (x1 - x0) * (y1 - y0)
        pos = starts[lane]
        if area <= COOP_AREA:
            tiles = [(y0 + b // w) * TILES_X + x0 + b % w for b in range(area) if (int(masks[lane]) >> b) & 1]
        else:
            tiles = big_tiles(lane)
        for tile in tiles:
            if pos < end:
                keys[pos] = tile
                vals[pos] = payloads[lane]
            pos += 1
    if total is not None:
        keys[min(total, end):end] = SENTINEL
        vals[min(total, end):end] = 0


def test_nth_set_bit():
    rng = np.random.RandomState(1)
    for _ in range(2000):
        m = int(rng.randint(1, 2**32, dtype=np.uint64))
        bits = [b for b in range(32) if (m >> b) & 1]
        for k, b in enumerate(bits):
            assert nth_set_bit(m, k) == b


def test_depth_order_emit_equals_per_lane_loops():
    rng = np.random.RandomState(0)
    for trial in range(400):
        kind = trial % 5
        x0 = rng.randint(0, 8, 32)
        y0 = rng.randint(0, 8, 32)
        w = rng.randint(1, 9, 32)
        h = rng.randint(1, 5, 32)
        if kind == 1:
            w[rng.rand(32) < 0.2] = 12                    # AABBs above COOP_AREA: the warp-wide test
        if kind == 2:
            w[:] = 32
            h[:] = 1                                      # full 32-bit masks
        bbs = np.stack([x0, y0, x0 + w, y0 + h], 1)
        area = w * h
        masks = np.array([int(rng.randint(0, 2**32, dtype=np.uint64)) & ((1 << min(a, 32)) - 1) if a <= COOP_AREA else 0
                          for a in area], dtype=np.uint64)
        if kind == 3:
            masks[rng.rand(32) < 0.5] = 0                 # visible rows that reach no tile
        big = {l: sorted(rng.choice(area[l], rng.randint(0, area[l] + 1), replace=False)) for l in range(32) if area[l] > COOP_AREA}
        big_tiles = lambda l: [(y0[l] + t // w[l]) * TILES_X + x0[l] + t % w[l] for t in big[l]]  # noqa: E731
        counts = np.array([bin(int(masks[l])).count("1") if area[l] <= COOP_AREA else len(big[l]) for l in range(32)])
        if kind == 4:
            counts[rng.randint(0, 32):] = 0               # invisible rows: last in depth order, nothing to emit
            masks[counts == 0] = 0
        first = rng.randint(0, 50)                        # the warp's first run starts behind earlier warps' entries
        starts = first + np.concatenate([[0], np.cumsum(counts)[:-1]])
        payloads = rng.randint(0, 2**31, 32) | np.where(rng.rand(32) < 0.3, -(2**31), 0)
        total = int(starts[-1] + counts[-1])
        capped = trial % 2 == 1
        end = int(rng.randint(first, total + 40)) if capped else total   # capacity below or above the count
        size = max(end, total) + 8
        got_k, got_v = np.full(size, -1, np.int64), np.full(size, -1, np.int64)
        want_k, want_v = got_k.copy(), got_v.copy()
        emulated(starts, counts, masks, bbs, payloads, big_tiles, end, total if capped else None, got_k, got_v)
        per_lane(starts, masks, bbs, payloads, big_tiles, end, total if capped else None, want_k, want_v)
        assert np.array_equal(got_k, want_k), trial
        assert np.array_equal(got_v, want_v), trial
        written = want_k[first:end] >= 0
        assert written.all(), trial                       # every slot below the end gets an entry or the padding
