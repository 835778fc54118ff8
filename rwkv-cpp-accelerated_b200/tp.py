"""Tensor-parallel plumbing: one process per GPU, `torch.distributed` only to swap the 64-byte CUDA IPC
handles of the ranks' exchange blocks at start-up. The data path has no collective call: the token kernel
stores its partial sums straight into the peers' exchange blocks over NVLink as self-tagged words
(csrc/exchange.cuh) and every rank reads only its own memory.

The split (SURVEY 8e, csrc/common.cuh `Params`): rank g of G owns the att channels and ffn key channels
[g*E/G, (g+1)*E/G) resp. [g*4E/G, (g+1)*4E/G): K, V, R, ffn-R and ffn-K are split by OUTPUT channel (columns of
the file's [in][out] layout), out-proj and ffn-V by INPUT channel (rows), the head by vocabulary row; the
loader reads only those slices. Residual stream, layernorm and token shift are replicated."""


def shard(n, world, rank):
    """[lo, hi) of a dimension of size n owned by `rank` - the arithmetic of engine.cu (do_load)."""
    return (n * rank) // world, (n * (rank + 1)) // world


def cta_slices(n_embed, world, rank, grid=132, vocab=50277):
    """Per-CTA row ranges inside rank `rank`'s shards - the arithmetic of make_slices() in csrc/token_kernel.cuh.
    Returns four lists of (first, count): residual elements (global, identical on every rank), att channels,
    ffn key channels and vocabulary rows (the last three relative to the rank's shard)."""
    er = n_embed // world
    v0, v1 = shard(vocab, world, rank)

    def split(m):
        return [((m * b) // grid, (m * (b + 1)) // grid - (m * b) // grid) for b in range(grid)]
    return split(n_embed), split(er), split(4 * er), split(v1 - v0)


def ffn_v_tiling(n_embed, world):
    """(segments per ffn-V row, rows per tile, bytes per tile) on one rank - the arithmetic of `Params::vseg`
    (engine.cu) and `load_sub` / `consume_sub` (csrc/token_kernel.cuh). A rank's ffn-V rows are 4E/G bytes; they are
    cut into 4, 2, 1 segments of at most E bytes for G = 1, 2, >= 4, and a tile (eight warp units) is 8 / segments rows."""
    seg = 1 if world >= 4 else 2 if world >= 2 else 4
    rows = 8 // seg
    return seg, rows, rows * (4 * n_embed // world)


def weight_bytes_per_rank(n_layers, n_embed, world, rank, vocab=50277):
    """uint8 weight bytes rank `rank` streams per token: 13 L E^2 / G + its vocabulary rows."""
    v0, v1 = shard(vocab, world, rank)
    return 13 * n_layers * n_embed * (n_embed // world) + (v1 - v0) * n_embed


def exchange_handles(handle, group=None):
    """All-gather one bytes object per rank, in rank order, over `group` (default: a gloo group created
    next to the default one - object collectives on NCCL need a CUDA context per pickle)."""
    import torch.distributed as dist
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    if group is None:
        group = dist.new_group(backend="gloo")
    out = [None] * dist.get_world_size(group)
    dist.all_gather_object(out, bytes(handle), group=group)
    return out


def connect(engine, group=None):
    """Wire a tensor-parallel Engine with its peers: export, all-gather, import."""
    import torch.distributed as dist
    handles = exchange_handles(engine.tp_export(), group)
    if len(handles) != engine.tp_size:
        raise RuntimeError("process group has %d ranks, engine expects %d" % (len(handles), engine.tp_size))
    engine.tp_import(handles)
    dist.barrier(group=group) if group is not None else dist.barrier()
