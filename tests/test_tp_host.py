"""Host side of the tensor-parallel path on CPU: the shard / slice arithmetic of the column-row split and
the handle exchange over a world-size-2 gloo group (no GPU, no compute calls)."""
import importlib
import os
import sys

import pytest

from util import ROOT


@pytest.fixture(scope="module")
def tp():
    sys.path.insert(0, ROOT)
    return importlib.import_module("rwkv-cpp-accelerated_b200").tp


@pytest.mark.parametrize("n_embed", [768, 2048, 4096, 5120])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_shards_and_slices_cover_everything_once(tp, n_embed, world):
    """Every att channel, ffn key channel and vocabulary row belongs to exactly one (rank, CTA); the residual
    slices are the same on every rank; the per-rank weight bytes add up to the whole model."""
    grid, vocab, L = 132, 50277, 3
    seen_c, seen_k, seen_v = [], [], []
    for rank in range(world):
        c0, c1 = tp.shard(n_embed, world, rank)
        assert c1 - c0 == n_embed // world
        k0, _ = tp.shard(4 * n_embed, world, rank)
        v0, v1 = tp.shard(vocab, world, rank)
        res, chan, keys, voc = tp.cta_slices(n_embed, world, rank, grid, vocab)
        assert res == tp.cta_slices(n_embed, world, 0, grid, vocab)[0]
        for lst, total in ((res, n_embed), (chan, n_embed // world), (keys, 4 * n_embed // world), (voc, v1 - v0)):
            assert lst[0][0] == 0 and sum(n for _, n in lst) == total
            assert all(a + n == b for (a, n), (b, _) in zip(lst, lst[1:]))   # contiguous, ascending
            assert max(n for _, n in lst) - min(n for _, n in lst) <= 1      # balanced to one row
        assert max(n for _, n in res) <= 64 and max(n for _, n in keys) <= 160  # kMaxSlice / kMaxKeys of the kernel
        seen_c += [c0 + a + i for a, n in chan for i in range(n)]
        seen_k += [k0 + a + i for a, n in keys for i in range(n)]
        seen_v += [v0 + a + i for a, n in voc for i in range(n)]
    assert seen_c == list(range(n_embed)) and seen_k == list(range(4 * n_embed)) and seen_v == list(range(vocab))
    assert sum(tp.weight_bytes_per_rank(L, n_embed, world, r) for r in range(world)) == 13 * L * n_embed ** 2 + vocab * n_embed


@pytest.mark.parametrize("n_embed", [768, 2048, 4096, 5120])
@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_ffn_v_tiles_fit_the_ring_and_the_limb_registers(tp, n_embed, world):
    """A unit (one warp's share of a tile) is a row segment of at most E bytes - the limbs of E bytes are what a warp
    holds in registers - and a tile never exceeds the ring stage of 8 x E bytes; up to four ranks it fills it."""
    seg, rows, tile = tp.ffn_v_tiling(n_embed, world)
    row_bytes = 4 * n_embed // world
    assert seg * rows == 8
    assert row_bytes % seg == 0 and row_bytes // seg <= n_embed
    assert tile <= 8 * n_embed
    if world <= 4:
        assert tile == 8 * n_embed


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    tp = importlib.import_module("rwkv-cpp-accelerated_b200").tp
    got = tp.exchange_handles(bytes([rank]) * 64, group=dist.group.WORLD)
    q.put((rank, got))
    dist.barrier()
    dist.destroy_process_group()


def test_handle_exchange_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, 29611, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in (0, 1):
        assert res[r] == [bytes([0]) * 64, bytes([1]) * 64]   # rank order, identical on every rank


def test_tp_load_needs_a_gpu_and_valid_rank():
    pkg = importlib.import_module("rwkv-cpp-accelerated_b200")
    lib = pkg.load_library()
    import ctypes
    h = ctypes.c_void_p()
    L, E = ctypes.c_ulonglong(), ctypes.c_ulonglong()
    rc = lib.rwkv_b200_load_tp(b"/nonexistent.bin", 1, 0, 1, 3, 2, ctypes.byref(h), ctypes.byref(L), ctypes.byref(E))
    assert rc != 0 and b"rank 3 of 2" in lib.rwkv_b200_last_error()
    assert lib.rwkv_b200_tp_buffer_bytes(None) == 0
