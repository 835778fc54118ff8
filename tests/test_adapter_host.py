"""LoRA adapters on the CPU: the C declarations, the key parser and its refusals, convert_model.py --lora against a
hand-merged checkpoint, and the float64 restatement's delta against a projection whose matrix has the adapter merged."""
import importlib.util
import os
import re

import numpy as np
import pytest
import torch

import lora_numerics as lm
import numerics as nm
from util import INCLUDE, ROOT

HEADER = open(os.path.join(INCLUDE, "rwkv_b200.h")).read()


def test_symbols_declared(pkg):
    for sym in ("rwkv_b200_adapter_add", "rwkv_b200_adapter_remove", "rwkv_b200_slot_adapter"):
        assert re.search(r"\bint %s\(" % sym, HEADER)
    assert "#define RWKV_B200_MAX_ADAPTER_RANK 64" in HEADER
    assert "#define RWKV_B200_NO_ADAPTER 0xFFFFFFFFFFFFFFFFULL" in HEADER
    lib = pkg.engine.load_library()
    assert lib.rwkv_b200_abi_version() == 2
    assert {"rwkv_b200_adapter_add", "rwkv_b200_adapter_remove", "rwkv_b200_slot_adapter"} <= set(lib._declared)
    for k, name in enumerate(pkg.engine.ADAPTER_MATRICES):
        macro = "RWKV_B200_AD_" + name.replace(".", "_").upper()
        assert "#define %s %d" % (macro, k) in HEADER


def lora(L, E, r, names=("att.key", "ffn.value"), seed=0):
    rng = np.random.default_rng(seed)
    w = {}
    for l in range(L):
        for n in names:
            ni = 4 * E if n == "ffn.value" else E
            no = 4 * E if n == "ffn.key" else E
            w["blocks.%d.%s.lora_A" % (l, n)] = rng.standard_normal((r, ni)).astype(np.float32)
            w["blocks.%d.%s.lora_B" % (l, n)] = rng.standard_normal((no, r)).astype(np.float32)
    return w


def test_parser(pkg):
    parse = pkg.engine.parse_adapter
    L, E = 2, 16
    rank, mats = parse(lora(L, E, 4), L, E)
    assert rank == 4 and set(mats) == {"att.key", "ffn.value"}
    assert mats["ffn.value"][0].shape == (L, 4, 4 * E) and mats["ffn.value"][1].shape == (L, E, 4)
    part = {k: v for k, v in lora(L, E, 4).items() if k.startswith("blocks.1.")}
    assert not parse(part, L, E)[1]["att.key"][0][0].any()        # a layer without the projection gets zeros
    bad = [
        ({"blocks.0.att.time_mix_k": np.zeros(E)}, "time_mix_k.*convert_model.py --lora"),
        ({"blocks.0.ln1.weight": np.zeros(E)}, "ln1.*convert_model.py --lora"),
        ({"blocks.0.att.key.lora_C": np.zeros((1, E))}, "lora_C"),
        ({"blocks.0.att.key.lora_A": np.zeros((2, E), np.float32)}, "no lora_B partner"),
        ({**lora(L, E, 4, ("att.key",)), **lora(L, E, 2, ("att.value",))}, "rank 2.*rank 4"),
        ({"blocks.0.att.key.lora_A": np.zeros((2, E + 1)), "blocks.0.att.key.lora_B": np.zeros((E, 2))}, "shape"),
        ({"blocks.0.att.key.lora_A": np.zeros((65, E)), "blocks.0.att.key.lora_B": np.zeros((E, 65))}, "rank 65"),
        ({"blocks.5.att.key.lora_A": np.zeros((2, E)), "blocks.5.att.key.lora_B": np.zeros((E, 2))}, "layer 5"),
        ({}, "no lora_A"),
    ]
    for w, msg in bad:
        with pytest.raises(ValueError, match=msg):
            parse(w, L, E)


@pytest.fixture(scope="module")
def conv():
    path = os.path.join(ROOT, "rwkv-cpp-accelerated_b200", "tools", "convert_model.py")
    spec = importlib.util.spec_from_file_location("convert_model_lora", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_convert_lora_equals_hand_merge(conv, tmp_path):
    L, E, r, alpha = 2, 64, 4, 8.0
    w = conv.synthetic_state_dict(L, E, 11)
    ad = {k: torch.from_numpy(v * 0.01) for k, v in lora(L, E, r, ("att.key", "att.output", "ffn.key", "ffn.value")).items()}
    ad["blocks.1.att.time_mix_k"] = torch.rand(1, 1, E, generator=torch.Generator().manual_seed(3))
    merged = dict(w)
    for k in ad:
        if k.endswith(".lora_A"):
            base = k[:-len(".lora_A")]
            B = ad[base + ".lora_B"].double()
            merged[base + ".weight"] = w[base + ".weight"].double() + (alpha / r) * (B @ ad[k].double())
    merged["blocks.1.att.time_mix_k"] = ad["blocks.1.att.time_mix_k"]
    paths = {n: str(tmp_path / n) for n in ("m.pth", "ad.pth", "h.pth", "a.bin", "b.bin")}
    torch.save(w, paths["m.pth"])
    torch.save(ad, paths["ad.pth"])
    torch.save(merged, paths["h.pth"])
    conv.convert(paths["m.pth"], paths["a.bin"], lora=paths["ad.pth"], lora_alpha=alpha)
    conv.convert(paths["h.pth"], paths["b.bin"])
    assert open(paths["a.bin"], "rb").read() == open(paths["b.bin"], "rb").read()
    plain = str(tmp_path / "p.bin")
    conv.convert(paths["m.pth"], plain)
    assert open(plain, "rb").read() != open(paths["a.bin"], "rb").read()
    with pytest.raises(ValueError, match="neither"):
        conv.merge_lora(w, {"blocks.0.att.nope": torch.zeros(1)}, 1.0)


@pytest.mark.parametrize("mode", ["exact", "engine"])
def test_restatement_without_adapters_is_numerics(make_model, mode):
    """lora_numerics with every stream unbound is numerics.forward (the same dataflow), and an adapter moves it."""
    from util import token_stream
    L, E = 2, 144
    model = nm.Model(make_model(L, E))
    streams = [token_stream(5, seed=1), token_stream(3, seed=2)]
    lg, st = lm.forward(model, streams, [None, None], mode=mode)
    rl, rs = nm.forward(model, streams, mode=mode)
    for a, b in zip(lg, rl):
        assert np.array_equal(a, b)
    for a, b in zip(st, rs):
        for k in nm.KEYS:
            assert np.array_equal(a[k], b[k]), k
    rng = np.random.default_rng(3)
    ad = {"scale": 2.0, "A": {"ffn_v": rng.standard_normal((L, 4, 4 * E)) * 0.05},
          "B": {"ffn_v": rng.standard_normal((L, E, 4)) * 0.05}}
    la, _ = lm.forward(model, streams, [ad, None], mode=mode)
    assert nm.logits_err(la[0], rl[0]) > 1e-3 and np.array_equal(la[1], rl[1])


def test_restatement_delta_is_a_merged_projection():
    """lora_numerics' delta, in exact mode, is the f64 projection through dequant(W) + s * B @ A, to a few f32 ulps."""
    rng = np.random.default_rng(1)
    N, M, T, r, s = 96, 80, 5, 8, 0.75
    w = rng.integers(0, 256, size=(N, M)).astype(np.uint8)
    rs, o = rng.random(N).astype(np.float32) * 0.01, (rng.standard_normal(N) * 0.1).astype(np.float32)
    f = rng.standard_normal((T, N)).astype(np.float32)
    A = rng.standard_normal((2, r, N)).astype(np.float32) * 0.1
    B = rng.standard_normal((2, M, r)).astype(np.float32) * 0.1
    ad = {"scale": s, "A": {"k": A}, "B": {"k": B}}
    d = lm.adapter_delta(ad, "k", 1, f)
    assert lm.adapter_delta(ad, "v", 1, f) is None and lm.adapter_delta(None, "k", 1, f) is None
    got = lm.project(f, w, rs, o, "exact", delta=d)
    W = w.astype(np.float64) * rs.astype(np.float64)[:, None] + o.astype(np.float64)[:, None]     # [in][out]
    W += s * (B[1].astype(np.float64) @ A[1].astype(np.float64)).T
    want = (f.astype(np.float64) @ W).astype(np.float32)
    ulp = np.spacing(np.abs(want))
    assert np.all(np.abs(got.astype(np.float64) - want) <= 4 * ulp)
    assert np.abs(got - nm.project(f, w, rs, o, "exact")).max() > 100 * ulp.max()
