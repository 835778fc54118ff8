"""The token kernel's producer fills each ring stage with bulk copies of at most `sub_bytes` (csrc/token_kernel.cuh,
produce_token: copy k of a tile of `bytes` covers [k * sub, k * sub + min(sub, bytes - k * sub))). For every tile of a
CTA's schedule - each sub of a layer, ffn V in 4, 2 or 1 segments per row, the head with its tail tile - and every
copy size the engine accepts, the copies must start 16-byte aligned, be multiples of 16 bytes, stay inside the stage
and add up to the tile, ceil(bytes / sub) of them."""
import importlib
import sys

import pytest

from util import ROOT

GRID = 132
VOCAB = 50277


@pytest.fixture(scope="module")
def tp():
    sys.path.insert(0, ROOT)
    return importlib.import_module("rwkv-cpp-accelerated_b200").tp


def copies(nbytes, sub):
    """(offset, size) of the bulk copies that fill one stage, in the producer's order."""
    out, off = [], 0
    while off < nbytes:
        n = min(sub, nbytes - off)
        out.append((off, n))
        off += n
    return out


def schedule_tiles(tp, n_embed, world, rank, cta):
    """Byte counts of the tiles one CTA streams per layer and for the head (load_sub / next_tile)."""
    er = n_embed // world
    res, chan, keys, voc = tp.cta_slices(n_embed, world, rank, GRID, VOCAB)
    seg, rows_v, _ = tp.ffn_v_tiling(n_embed, world)
    subs = [(chan[cta][1], n_embed, 8)] * 3 + [(res[cta][1], er, 8), (keys[cta][1], n_embed, 8),
                                                (chan[cta][1], n_embed, 8), (res[cta][1], 4 * er, rows_v)]
    tiles = []
    for nr, row_bytes, tr in subs + [(voc[cta][1], n_embed, 8)]:
        tiles += [min(tr, nr - r) * row_bytes for r in range(0, nr, tr)]
    return tiles


# ffn V in 4, 2, 1 segments per row on 1, 2, 4 ranks (n_embed / ranks a multiple of 16)
@pytest.mark.parametrize("n_embed,world", [(144, 1), (784, 1), (768, 1), (768, 2), (768, 4), (4096, 1), (4096, 2),
                                           (4096, 4), (5120, 1), (5120, 2), (5120, 4)])
def test_stage_copies_cover_every_tile(tp, n_embed, world):
    tile_bytes = 8 * n_embed
    subs = sorted({16, 1024, 4096, 8192, 16384, tile_bytes // 3 // 16 * 16, tile_bytes - 16, tile_bytes})
    subs = [s for s in subs if 16 <= s <= tile_bytes]
    seen_tail = False
    for cta in (0, 1, GRID // 2, GRID - 1):
        tiles = schedule_tiles(tp, n_embed, world, 0, cta)
        seen_tail |= any(b < tile_bytes for b in tiles)
        for nbytes in set(tiles):
            assert 0 < nbytes <= tile_bytes and nbytes % 16 == 0, (cta, nbytes)
            for sub in subs:
                cs = copies(nbytes, sub)
                assert len(cs) == -(-nbytes // sub)
                assert sum(n for _, n in cs) == nbytes
                assert all(off % 16 == 0 and n % 16 == 0 and 0 < n <= sub for off, n in cs)
                assert cs[-1][0] + cs[-1][1] <= tile_bytes
    assert seen_tail  # the head's last tile (and narrow slices) are shorter than a stage


def test_head_tail_tile():
    """50277 vocabulary rows over 132 CTAs: 380 or 381 rows each, so every CTA ends its head on a partial tile."""
    n_embed, sub = 4096, 8192
    rows = [(VOCAB * (b + 1)) // GRID - (VOCAB * b) // GRID for b in range(GRID)]
    assert set(rows) == {380, 381}
    for nr in set(rows):
        tail = (nr % 8) * n_embed
        assert 0 < tail < 8 * n_embed
        assert [n for _, n in copies(tail, sub)] == [sub] * (tail // sub) + ([tail % sub] if tail % sub else [])
