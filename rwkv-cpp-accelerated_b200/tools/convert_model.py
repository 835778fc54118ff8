"""RWKV-4 `.pth` checkpoint -> reference-format uint8 `.bin` (SURVEY §8f N2), written from scratch.

Produces byte-for-byte what the reference's converter produces (converter/convert_model.py:14-176 builds
the tensors, converter/cpp_save_tensor.cpp:75-95 writes them) without its torch C++ extension:
    python convert_model.py model.pth [model.bin] [--lora adapter.pth --lora-alpha A]

--lora merges a LoRA fine-tune into the weights before quantising (merge_lora): the fast path for one fine-tune on one
stream, since the decode kernel then runs it at full speed. Several fine-tunes of one base model served together bind
runtime adapters to state slots instead (Engine.add_adapter).

File layout (include/rwkv/rwkv/format.h is the table this follows): two little-endian int64
{n_layers, n_embed}, then the 46 tensors in enum order, unpadded - including the scratch buffers and the
zero / -1e30 state sections the engines ignore (convert_model.py:19-25, 99-106).

Q8 scheme (convert_model.py:108-119) for a Linear weight W[out][in]: per INPUT column j
    lo_j = min_out W, ran_j = (max_out W - lo_j) / 255, q = trunc((W - lo_j) / ran_j) in 0..255,
    zp_j = lo_j + mean_out(frac((W - lo_j) / ran_j)) * ran_j          (bias correction of the truncation)
stored transposed [in][out] uint8 with ranges[in], zp[in] as f32; all arithmetic in f64.
Pinned bit-exact against the reference's own Python class: tests/golden/converter_golden.json.
"""
import argparse
import struct

import numpy as np
import torch

VOCAB = 50277

# (name in the file table, dtype) in enum order - checked against format.h by tests/test_converter.py
ORDER = [
    ("xbuf", "f8"), ("embed", "f4"), ("layernorms", "f8"), ("state_xy", "f8"), ("state_aa", "f8"), ("state_bb", "f8"),
    ("state_pp", "f8"), ("state_dd", "f8"), ("buffer1", "f8"), ("buffer2", "f4"), ("buffer3", "f4"), ("buffer4", "f4"),
    ("mix_k", "f8"), ("mix_v", "f8"), ("mix_r", "f8"), ("km", "u1"), ("vm", "u1"), ("rm", "u1"), ("kr", "f4"),
    ("vr", "f4"), ("rr", "f4"), ("o1", "f4"), ("o2", "f4"), ("o3", "f4"), ("att_out", "u1"), ("att_out_r", "f4"),
    ("att_out_o", "f4"), ("ffn_mix_k", "f8"), ("ffn_mix_v", "f8"), ("ffn_k", "u1"), ("ffn_v", "u1"), ("ffn_r", "u1"),
    ("ffn_kr", "f4"), ("ffn_vr", "f4"), ("ffn_rr", "f4"), ("ffn_ko", "f4"), ("ffn_vo", "f4"), ("ffn_ro", "f4"),
    ("ffn_k_buffer", "f8"), ("ffn_v_buffer", "f8"), ("ffn_r_buffer", "f4"), ("decay", "f8"), ("bonus", "f8"),
    ("head", "u1"), ("head_r", "f4"), ("head_o", "f4"),
]


def quantize_matrix(w):
    """W[out][in] (any float dtype) -> (q [in][out] uint8, ranges [in] f32, zp [in] f32)."""
    x = w.to(torch.float64)
    lo = x.min(dim=0).values
    span = x - lo
    ran = span.max(dim=0).values / 255
    scaled = span / ran
    zp = lo + scaled.frac().mean(dim=0) * ran
    return scaled.t().to(torch.uint8).contiguous(), ran.to(torch.float32), zp.to(torch.float32)


def model_dims(w):
    n_embed = int(w["blocks.0.att.key.weight"].shape[0])
    n_layers = sum(1 for k in w if k.startswith("blocks.") and k.endswith("ln1.bias"))
    return n_layers, n_embed


def build_tensors(w):
    """state dict -> (n_layers, n_embed, dict name -> contiguous torch tensor of the file dtype)."""
    L, E = model_dims(w)
    out = {}

    def per_layer(fmt):
        return [w[fmt.format(i)] for i in range(L)]

    def vec64(fmt):
        return torch.stack([t.squeeze() for t in per_layer(fmt)]).to(torch.float64).contiguous()

    ln_names = ["blocks.0.ln0.weight", "blocks.0.ln0.bias"]
    for i in range(L):
        ln_names += ["blocks.%d.ln1.weight" % i, "blocks.%d.ln1.bias" % i, "blocks.%d.ln2.weight" % i, "blocks.%d.ln2.bias" % i]
    ln_names += ["ln_out.weight", "ln_out.bias"]

    out["xbuf"] = torch.arange(E, dtype=torch.float64)
    out["embed"] = w["emb.weight"].to(torch.float32).contiguous()
    out["layernorms"] = torch.stack([w[n] for n in ln_names]).to(torch.float64).contiguous()
    zeros = torch.zeros(L, E, dtype=torch.float64)
    out["state_xy"], out["state_aa"], out["state_bb"], out["state_dd"] = zeros, zeros, zeros, zeros
    # the reference builds its placeholder from a float32 tensor: the stored value is float32(-1e30) widened
    out["state_pp"] = torch.full((L, E), -1e30, dtype=torch.float32).to(torch.float64)
    out["buffer1"] = torch.arange(E, dtype=torch.float64)
    out["buffer2"] = torch.arange(VOCAB, dtype=torch.float32)
    out["buffer3"] = torch.arange(E, dtype=torch.float32)
    out["buffer4"] = torch.arange(E, dtype=torch.float32)
    out["mix_k"] = vec64("blocks.{}.att.time_mix_k")
    out["mix_v"] = vec64("blocks.{}.att.time_mix_v")
    out["mix_r"] = vec64("blocks.{}.att.time_mix_r")
    out["ffn_mix_k"] = vec64("blocks.{}.ffn.time_mix_k")
    out["ffn_mix_v"] = vec64("blocks.{}.ffn.time_mix_r")  # the file's "ffnmixv" slot holds time_mix_r (convert_model.py:55-56)
    out["decay"] = -torch.exp(vec64("blocks.{}.att.time_decay"))
    out["bonus"] = vec64("blocks.{}.att.time_first")

    def family(fmt, qn, rn, on):
        parts = [quantize_matrix(t) for t in per_layer(fmt)]
        out[qn] = torch.stack([p[0] for p in parts]).contiguous()
        out[rn] = torch.stack([p[1] for p in parts]).contiguous()
        out[on] = torch.stack([p[2] for p in parts]).contiguous()

    family("blocks.{}.att.key.weight", "km", "kr", "o1")
    family("blocks.{}.att.value.weight", "vm", "vr", "o2")
    family("blocks.{}.att.receptance.weight", "rm", "rr", "o3")
    family("blocks.{}.att.output.weight", "att_out", "att_out_r", "att_out_o")
    family("blocks.{}.ffn.key.weight", "ffn_k", "ffn_kr", "ffn_ko")
    family("blocks.{}.ffn.value.weight", "ffn_v", "ffn_vr", "ffn_vo")
    family("blocks.{}.ffn.receptance.weight", "ffn_r", "ffn_rr", "ffn_ro")
    out["ffn_k_buffer"] = torch.arange(E, dtype=torch.float64)
    out["ffn_v_buffer"] = torch.arange(E, dtype=torch.float64)
    out["ffn_r_buffer"] = torch.arange(4 * E, dtype=torch.float32)
    out["head"], out["head_r"], out["head_o"] = quantize_matrix(w["head.weight"])
    return L, E, out


def expected_elems(name, L, E):
    big = {"embed": VOCAB * E, "head": VOCAB * E, "layernorms": 4 * (L + 1) * E, "buffer2": VOCAB}
    if name in big:
        return big[name]
    if name in ("xbuf", "buffer1", "buffer3", "buffer4", "ffn_k_buffer", "ffn_v_buffer", "head_r", "head_o"):
        return E
    if name == "ffn_r_buffer":
        return 4 * E
    if name in ("km", "vm", "rm", "att_out", "ffn_r"):
        return L * E * E
    if name in ("ffn_k", "ffn_v"):
        return 4 * L * E * E
    if name in ("ffn_vr", "ffn_vo"):
        return 4 * L * E
    return L * E


def write_bin(path, L, E, tensors):
    np_dtype = {"f8": np.float64, "f4": np.float32, "u1": np.uint8}
    with open(path, "wb") as f:
        f.write(struct.pack("<qq", L, E))
        for name, dt in ORDER:
            a = tensors[name].contiguous().numpy()
            if a.dtype != np_dtype[dt] or a.size != expected_elems(name, L, E):
                raise ValueError("tensor %s: dtype %s / %d elements, expected %s / %d"
                                 % (name, a.dtype, a.size, dt, expected_elems(name, L, E)))
            f.write(a.tobytes())


def merge_lora(w, lora, alpha):
    """The state dict w with a LoRA fine-tune merged in. Each pair "<linear>.lora_A" [r][in] / "<linear>.lora_B"
    [out][r] (the RWKV-4 LoRA trainers' naming) adds s * B @ A, s = alpha / r, to "<linear>.weight" in float64; any other
    key of `lora` that the checkpoint has (the trainers' full-parameter time_* and ln tensors) replaces it. Unknown
    keys, a missing partner and wrong shapes raise ValueError."""
    w = dict(w)
    for key, val in lora.items():
        if key.endswith(".lora_A") or key.endswith(".lora_B"):
            base = key[:-len(".lora_A")]
            if base + ".weight" not in w:
                raise ValueError("LoRA key %s: the checkpoint has no %s.weight" % (key, base))
            if key.endswith(".lora_B"):
                continue
            if base + ".lora_B" not in lora:
                raise ValueError("LoRA key %s has no lora_B partner" % key)
            A, B = val.to(torch.float64), lora[base + ".lora_B"].to(torch.float64)
            W = w[base + ".weight"]
            if A.dim() != 2 or B.dim() != 2 or B.shape[1] != A.shape[0] or (B.shape[0], A.shape[1]) != tuple(W.shape):
                raise ValueError("LoRA %s: A %s and B %s do not fit the weight %s" % (base, tuple(A.shape), tuple(B.shape),
                                                                                     tuple(W.shape)))
            w[base + ".weight"] = W.to(torch.float64) + (alpha / A.shape[0]) * (B @ A)
        elif key in w:
            if tuple(val.shape) != tuple(w[key].shape):
                raise ValueError("LoRA key %s has shape %s, the checkpoint's has %s" % (key, tuple(val.shape), tuple(w[key].shape)))
            w[key] = val
        else:
            raise ValueError("LoRA key %s is neither a lora_A / lora_B pair nor a tensor of the checkpoint" % key)
    for key in lora:
        if key.endswith(".lora_B") and key[:-len(".lora_B")] + ".lora_A" not in lora:
            raise ValueError("LoRA key %s has no lora_A partner" % key)
    return w


def convert(pth_path, bin_path, lora=None, lora_alpha=None):
    w = torch.load(pth_path, map_location="cpu")
    for k in ("emb.weight", "ln_out.weight", "ln_out.bias", "blocks.0.ln0.weight", "blocks.0.ln0.bias", "head.weight"):
        if k not in w:
            raise ValueError("not an RWKV-4 checkpoint: missing %s" % k)
    if lora is not None:
        if lora_alpha is None:
            raise ValueError("--lora needs --lora-alpha")
        w = merge_lora(w, torch.load(lora, map_location="cpu"), float(lora_alpha))
    L, E, tensors = build_tensors(w)
    print("n_layers %d  n_embed %d" % (L, E))
    write_bin(bin_path, L, E, tensors)
    return L, E


def synthetic_state_dict(L, E, seed, dtype=torch.float32):
    """A random RWKV-4 shaped state dict (tests and the golden generator share it)."""
    g = torch.Generator().manual_seed(seed)

    def rnd(*shape, scale=1.0):
        return (torch.randn(*shape, generator=g) * scale).to(dtype)

    w = {"emb.weight": rnd(VOCAB, E, scale=0.1), "head.weight": rnd(VOCAB, E, scale=E ** -0.5),
         "ln_out.weight": 1 + rnd(E, scale=0.1), "ln_out.bias": rnd(E, scale=0.1),
         "blocks.0.ln0.weight": 1 + rnd(E, scale=0.1), "blocks.0.ln0.bias": rnd(E, scale=0.1)}
    for i in range(L):
        b = "blocks.%d." % i
        for ln in ("ln1", "ln2"):
            w[b + ln + ".weight"] = 1 + rnd(E, scale=0.1)
            w[b + ln + ".bias"] = rnd(E, scale=0.1)
        for m in ("att.time_mix_k", "att.time_mix_v", "att.time_mix_r", "ffn.time_mix_k", "ffn.time_mix_r"):
            w[b + m] = torch.rand(1, 1, E, generator=g).to(dtype)
        w[b + "att.time_decay"] = rnd(E)
        w[b + "att.time_first"] = rnd(E, scale=0.5)
        for m in ("att.key", "att.value", "att.receptance", "att.output", "ffn.receptance"):
            w[b + m + ".weight"] = rnd(E, E, scale=E ** -0.5)
        w[b + "ffn.key.weight"] = rnd(4 * E, E, scale=E ** -0.5)
        w[b + "ffn.value.weight"] = rnd(E, 4 * E, scale=(4 * E) ** -0.5)
    return w


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("pth")
    ap.add_argument("bin", nargs="?", default="model.bin")
    ap.add_argument("--lora", help="a LoRA checkpoint to merge before quantising")
    ap.add_argument("--lora-alpha", type=float, help="the LoRA alpha: the scale is alpha / rank")
    a = ap.parse_args()
    convert(a.pth, a.bin, a.lora, a.lora_alpha)
