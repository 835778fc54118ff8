"""The token kernel's launch geometry, restated on the host: which grids csrc/engine.cu grid_fits admits, what each CTA of
such a grid then owns (csrc/token_kernel.cuh make_slices), and whether that fits everything the kernel holds per CTA.

The engine runs one CTA per SM by default and takes any other grid through set_option("grid", n); a GPU with another SM
count (114 on an H100 PCIe) runs another one too. Every grid grid_fits admits must keep each CTA inside the kernel's
per-CTA arrays and thread roles, for every width the loader accepts: a grid that breaks one would write past a shared
array or leave an element without an owner, with no error at the launch.

Also here: the grids tests/test_grid_gpu.py must visit per width (the smallest admitted grid, the grids that give a CTA
the most residual elements, ffn keys and vocabulary rows, an odd grid with uneven slices, the H100 PCIe's 114 and the
default), the ring depths it must run, and the default ring depth of every width (csrc/engine.cu configure_ring)."""
import os
import re

import pytest

import numerics as nm
import test_grid_gpu as gpu
from util import PKG_DIR

CSRC = os.path.join(PKG_DIR, "csrc")
V = nm.V
DEFAULT_GRID = 132   # SMs of an H100 SXM
PCIE_GRID = 114      # SMs of an H100 PCIe
WIDTHS = range(16, 5121, 16)  # every n_embed the loader accepts (engine.cu do_load)


def source(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def flat(text):
    return re.sub(r"\s+", " ", text)


def constant(name):
    m = re.search(r"constexpr int %s = (\d+);" % name, source("common.cuh"))
    assert m, "%s not found in csrc/common.cuh" % name
    return int(m.group(1))


K = {n: constant(n) for n in ("kMaxGrid", "kMaxSlice", "kMaxKeys", "kMaxRowsPerCta", "kMaxStages", "kSmemLimit", "kWarps")}
CONSUMERS = 32 * K["kWarps"]


# -- the restatements -----------------------------------------------------------------------------------------------

def split(m, grid):
    """(first, count) of CTA b for b in 0..grid-1: split_rows in csrc/token_kernel.cuh."""
    return [((m * b) // grid, (m * (b + 1)) // grid - (m * b) // grid) for b in range(grid)]


def counts(E, grid, world=1, rank=0):
    """The largest count over the CTAs of each slice (make_slices): residual elements ne, att channels nc, ffn key
    channels nk, vocabulary rows nv."""
    er = E // world
    v0, v1 = (V * rank) // world, (V * (rank + 1)) // world
    big = lambda m: max(n for _, n in split(m, grid))
    return {"ne": big(E), "nc": big(er), "nk": big(4 * er), "nv": big(v1 - v0)}


def grid_fits(E, Er, Vr, grid):
    """csrc/engine.cu grid_fits."""
    up = lambda a: -(-a // grid) + 1
    ne, nc, nk, nv = up(E), up(Er), up(4 * Er), up(Vr)
    return (1 <= grid <= K["kMaxGrid"] and E >= grid and ne <= K["kMaxSlice"] and nk <= 160 and nk + nc <= K["kMaxRowsPerCta"]
            and 4 * ne <= K["kMaxRowsPerCta"] and 3 * nc <= K["kMaxRowsPerCta"] and nv <= K["kMaxRowsPerCta"])


def admitted(E, world=1, rank=0):
    Vr = (V * (rank + 1)) // world - (V * rank) // world
    return [g for g in range(1, K["kMaxGrid"] + 1) if grid_fits(E, E // world, Vr, g)]


def kernel_limits(E, grid, world=1, rank=0):
    """Every per-CTA capacity of csrc/token_kernel.cuh and common.cuh at this geometry: a list of (what, need, have)."""
    c = counts(E, grid, world, rank)
    ne, nc, nk, nv = c["ne"], c["nc"], c["nk"], c["nv"]
    vseg = 1 if world >= 4 else 2 if world >= 2 else 4   # segments per ffn-V row (engine.cu, Params::vseg)
    rows = K["kMaxRowsPerCta"]
    # publish_slice keeps the parts of warps 1..nw-1 in scal[10..15]: (nw - 1) * NV <= 6 doubles
    scratch = lambda n, nv_: (max(-(-n // 32), 1) - 1) * nv_
    return [
        ("grid <= kMaxGrid (slice_stats reads kMaxGrid / 32 records per lane)", grid, K["kMaxGrid"]),
        ("grid <= records a gather reads (one per consumer thread)", grid, CONSUMERS),
        ("ne <= kMaxSlice (xown, pd, pf; owners are warps 0 and 1; slice_stats sums lane and lane + 32)", ne, K["kMaxSlice"]),
        ("nc <= kMaxSlice (WKV and sigmoid(ffn r) owners in warps 0 and 1, srown)", nc, K["kMaxSlice"]),
        ("nk <= kMaxKeys (pk: ffn-V scale and offset of the own keys)", nk, K["kMaxKeys"]),
        ("nk <= consumer threads (one thread per own key channel)", nk, CONSUMERS),
        ("res64: K, V, R totals (3 nc)", 3 * nc, rows),
        ("res64: ffn-R then ffn-K totals (nc + nk)", nc + nk, rows),
        ("res64: out-proj totals (ne)", ne, rows),
        ("res64: ffn-V segment totals (vseg ne)", vseg * ne, rows),
        ("res64: head totals (nv)", nv, rows),
        ("publish_slice scratch: xk, xv, xr of ne elements", scratch(ne, 3), 6),
        ("publish_slice scratch: ffn xr, xk of ne elements", scratch(ne, 2), 6),
        ("publish_slice scratch: head input of ne elements", scratch(ne, 1), 6),
        ("publish_slice scratch: att out input of nc channels", scratch(nc, 1), 6),
        ("publish_slice scratch: relu^2 of nk keys", scratch(nk, 1), 6),
    ]


def smem_fixed_bytes():
    """csrc/common.cuh smem_fixed_bytes."""
    return (K["kMaxRowsPerCta"] * 8 + 16 * 8 + K["kWarps"] * 4 * 4 + 2 * K["kMaxStages"] * 8 + K["kMaxSlice"] * (8 + 4 + 64 + 32)
            + K["kMaxKeys"] * 8 + 128 + 16 + K["kWarps"] * 3 * 8)


def smem_bytes(stages, E):
    """csrc/common.cuh smem_bytes for the ring of an n_embed = E model: tiles of 8 E bytes, 12 E bytes of limb planes."""
    return stages * 8 * E + 12 * E + smem_fixed_bytes()


def max_stages(E):
    """The deepest ring set_option("stages") accepts, which is also configure_ring's default."""
    return min(K["kMaxStages"], (K["kSmemLimit"] - smem_bytes(0, E)) // (8 * E))


def uneven(E, grid):
    return E % grid and (4 * E) % grid and V % grid


def grids_to_visit(E, sms=DEFAULT_GRID):
    """The grids tests/test_grid_gpu.py must run at width E: the smallest admitted grid, the smallest grid with the
    largest ne, nk and nv each, an odd grid with every slice uneven (the one nearest the middle of the smallest admitted
    grid and the default), the H100 PCIe's 114 where it is admitted, and the default. None above `sms`."""
    ok = [g for g in admitted(E) if g <= sms]
    need = {ok[0], sms}
    for key in ("ne", "nk", "nv"):
        top = max(counts(E, g)[key] for g in ok)
        need.add(min(g for g in ok if counts(E, g)[key] == top))
    mid = (ok[0] + sms) / 2
    need.add(min((g for g in ok if g % 2 and uneven(E, g)), key=lambda g: (abs(g - mid), g)))
    if PCIE_GRID in ok:
        need.add(PCIE_GRID)
    return sorted(need)


def stages_to_visit(E):
    """Ring depths tests/test_grid_gpu.py must run: 2, 3, the odd depth nearest the middle of 2..max_stages, and
    max_stages."""
    top = max_stages(E)
    odd = min((s for s in range(3, top + 1, 2)), key=lambda s: (abs(s - (2 + top) / 2), s))
    return sorted({2, 3, odd, top})


# -- the restatements are the engine's --------------------------------------------------------------------------------

def test_restated_arithmetic_is_the_engines():
    eng, tk, common = flat(source("engine.cu")), flat(source("token_kernel.cuh")), flat(source("common.cuh"))
    bodies = {
        "engine.cu grid_fits": (eng, "const unsigned long long ne = (E + g - 1) / g + 1, nc = (Er + g - 1) / g + 1, nk = "
                                "(4 * Er + g - 1) / g + 1, nv = (Vr + g - 1) / g + 1; return grid >= 1 && grid <= "
                                "rk::kMaxGrid && E >= g && ne <= (unsigned long long)rk::kMaxSlice && nk <= 160 && nk + nc "
                                "<= (unsigned long long)rk::kMaxRowsPerCta && 4 * ne <= (unsigned long long)rk::kMaxRowsPerCta "
                                "&& 3 * nc <= (unsigned long long)rk::kMaxRowsPerCta && nv <= (unsigned long long)"
                                "rk::kMaxRowsPerCta; }"),
        "engine.cu configure_ring": (eng, "p.tile_bytes = (int)(8 * m->E); p.stages = (int)std::min<size_t>(rk::kMaxStages, "
                                     "(rk::kSmemLimit - rk::smem_bytes(0, 0, p.plane_cap)) / p.tile_bytes);"),
        "engine.cu plane_cap": (eng, "p.plane_cap = (int)(12 * E);"),
        "engine.cu set_option stages": (eng, "const size_t smem = rk::smem_bytes(v, m->p.tile_bytes, m->p.plane_cap); if "
                                        "(smem > (size_t)rk::kSmemLimit)"),
        "token_kernel.cuh split_rows": (tk, "r0 = (int)(((unsigned int)M * (unsigned int)b) / (unsigned int)nb); n = (int)"
                                        "(((unsigned int)M * (unsigned int)(b + 1)) / (unsigned int)nb) - r0;"),
        "token_kernel.cuh make_slices": (tk, "split_rows(E, b, nb, s.e0, s.ne); split_rows(Er, b, nb, s.c0, s.nc); "
                                         "split_rows(4 * Er, b, nb, s.k0, s.nk); split_rows(Vr, b, nb, s.v0, s.nv);"),
        "common.cuh smem_fixed_bytes": (common, "return kMaxRowsPerCta * 8 + 16 * 8 + kWarps * 4 * 4 + 2 * kMaxStages * 8 + "
                                        "kMaxSlice * (8 + 4 + 64 + 32) + kMaxKeys * 8 + 128 + 16 + kWarps * 3 * 8;"),
        "common.cuh smem_bytes": (common, "return (size_t)stages * tile_bytes + plane_cap + smem_fixed_bytes();"),
        "token_kernel.cuh publish_slice scratch": (tk, "double *scr = sm.scal + 10; // [nw - 1][NV] <= 6 doubles"),
        "common.cuh scal": (common, "double *scal; // [16]"),
    }
    stale = [what for what, (src, body) in bodies.items() if body not in src]
    assert not stale, "changed in csrc: restate them in tests/test_grid_host.py: %s" % stale
    # the split of tp.py, which the tensor-parallel tests use, is the same one
    import importlib
    tp = importlib.import_module("rwkv-cpp-accelerated_b200.tp")
    for E, g in ((768, 50), (5120, 129), (1040, 77)):
        assert list(tp.cta_slices(E, 1, 0, grid=g)) == [split(E, g), split(E, g), split(4 * E, g), split(V, g)]


def test_restated_counts_at_the_smallest_and_default_grids():
    """The ceilings of the even split at the smallest admitted grid and at 132 (one CTA per SM of an H100 SXM)."""
    want = {768: (50, (16, 62, 1006), (6, 24, 381)), 2048: (52, (40, 158, 967), (16, 63, 381)),
            4096: (104, (40, 158, 484), (32, 125, 381)), 5120: (129, (40, 159, 390), (39, 156, 381))}
    for E, (gmin, at_min, at_default) in want.items():
        assert admitted(E)[0] == gmin, E
        for g, trio in ((gmin, at_min), (DEFAULT_GRID, at_default)):
            c = counts(E, g)
            assert (c["ne"], c["nk"], c["nv"]) == trio, (E, g, c)


# -- every admitted grid fits the kernel --------------------------------------------------------------------------------

@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_every_admitted_grid_fits_the_kernel(world):
    """For every width and rank layout the loader accepts and every grid 1..kMaxGrid that grid_fits admits, each CTA
    stays within every per-CTA capacity of the kernel."""
    bad, checked = [], 0
    for E in WIDTHS:
        if E % (16 * world):
            continue
        for rank in range(world):
            for g in admitted(E, world, rank):
                checked += 1
                for what, need, have in kernel_limits(E, g, world, rank):
                    if need > have:
                        bad.append("E=%d G=%d rank %d grid %d: %s: %d > %d" % (E, world, rank, g, what, need, have))
    assert checked, world
    assert not bad, "grid_fits admits grids the token kernel cannot hold:\n" + "\n".join(bad[:20])


def test_default_grids_load():
    """One CTA per SM: the H100 SXM loads every width from 132 on; the H100 PCIe every width up to 4528 from 114 on.
    Wider models need a grid of more than 114 CTAs (the head rows of a CTA), so the loader refuses them there."""
    assert [E for E in WIDTHS if DEFAULT_GRID not in admitted(E)] == list(range(16, DEFAULT_GRID, 16))
    assert [E for E in WIDTHS if PCIE_GRID not in admitted(E)] == list(range(16, PCIE_GRID, 16)) + list(range(4544, 5121, 16))


def test_smallest_grids():
    """Print the smallest admitted grid and what a CTA owns there for the widths of the GPU grid tests."""
    for E in sorted(gpu.GRIDS):
        g = admitted(E)[0]
        c = counts(E, g)
        print("E=%d: grids %d..%d admitted; at %d a CTA owns up to ne %d nc %d nk %d nv %d" % (
            E, g, admitted(E)[-1], g, c["ne"], c["nc"], c["nk"], c["nv"]))
        # one grid fewer breaks a capacity grid_fits checks (the message the GPU test expects)
        assert not grid_fits(E, E, V, g - 1)


# -- the GPU file covers what it must ------------------------------------------------------------------------------------

def test_gpu_grid_lists_are_complete():
    widths = sorted({c["E"] for c in nm.cases() if c["path"] == "decode"} | {E for E in nm.WIDE if "decode" in nm.WIDE[E]})
    assert sorted(gpu.GRIDS) == widths, "tests/test_grid_gpu.py GRIDS: one entry per decode-kernel width of numerics"
    assert {E for _, _, E in gpu.CASES} == set(widths)
    for E in widths:
        need = grids_to_visit(E)
        have = gpu.GRIDS[E]
        missing = sorted(set(need) - set(have))
        assert not missing, "tests/test_grid_gpu.py GRIDS[%d] misses grids %s (needs %s)" % (E, missing, need)
        for g in have:
            assert g in admitted(E) and g <= DEFAULT_GRID, "GRIDS[%d]: %d is not an admitted grid" % (E, g)
        assert gpu.GRIDS[E][0] == admitted(E)[0], "GRIDS[%d] starts at the smallest admitted grid" % E


def test_gpu_case_streams_are_the_proven_ones(monkeypatch):
    """The tokens of every case are those numerics.inputs and numerics.depth_passes give it, which the host numerics
    tests prove mutation-sensitive. (depth_passes restates the ragged states of the 4096 group before it returns; that
    restatement is stubbed out here, since only the case streams are compared.)"""
    import types
    monkeypatch.setattr(nm, "forward", lambda model, streams, *a, **k: (None, [None] * len(streams)))
    for cid, L, E in gpu.CASES:
        case = [c for c in nm.cases() if c["id"] == cid]
        if case:
            assert gpu.case_stream(cid, L, E) == nm.inputs(case[0], None)[0][0], cid
        else:
            ids, streams, _ = nm.depth_passes(E, types.SimpleNamespace(L=L, E=E))[0]
            assert gpu.case_stream(cid, L, E) == streams[ids.index(cid)], cid


def test_gpu_option_lists_are_complete():
    for (L, E) in gpu.SHAPES.values():
        need = stages_to_visit(E)
        missing = sorted(set(need) - set(gpu.STAGES[E]))
        assert not missing, "tests/test_grid_gpu.py STAGES[%d] misses %s (needs %s)" % (E, missing, need)
        assert max(gpu.STAGES[E]) == max_stages(E)
        if max_stages(E) < K["kMaxStages"]:
            assert smem_bytes(max_stages(E) + 1, E) > K["kSmemLimit"]
            assert gpu.STAGES_OVER[E] == max_stages(E) + 1, "STAGES_OVER[%d]: the first depth above the limit" % E
        else:
            assert gpu.STAGES_OVER.get(E) is None
    assert {0, 1, 64} <= set(gpu.PF_DISTS)
    assert K["kMaxStages"] + 1 == 13  # the refusal the GPU file names


# -- the default ring depth ------------------------------------------------------------------------------------------------

def test_default_ring_depth():
    """configure_ring: as many stages of 8 E bytes as fit beside the limb planes and the fixed arrays, at most 12. Every
    width has room for two (the loader's floor); widths up to 1984 run all 12."""
    table = {E: max_stages(E) for E in WIDTHS}
    assert min(table.values()) >= 2
    assert all(table[a] >= table[b] for a, b in zip(WIDTHS, WIDTHS[1:]))
    runs = {}
    for E, s in table.items():
        runs.setdefault(s, []).append(E)
    print("default ring depth: " + "; ".join("%d stages: n_embed %d..%d" % (s, min(v), max(v)) for s, v in sorted(runs.items())))
    assert max(runs[K["kMaxStages"]]) == 1984
    assert [table[E] for E in (768, 2048, 2560, 3072, 4096, 5120)] == [12, 11, 9, 7, 5, 3]
    for E in WIDTHS:
        assert smem_bytes(table[E], E) <= K["kSmemLimit"]
        assert table[E] == K["kMaxStages"] or smem_bytes(table[E] + 1, E) > K["kSmemLimit"]
