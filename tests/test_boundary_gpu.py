"""The drop-in boundary on a real GPU (SURVEY 8b):

  * the reference's OWN, unmodified host header (rwkv.h:245-429) linked against this engine's
    implementation of its six backend hooks (include/rwkv/b200/rwkv_hooks.cpp): RWKV::loadFile +
    RWKV::forward through `oracle/_ref/ref_harness_b200`, logits and state checked against the oracle;
  * the reference's example program examples/storygen/storygen.cpp, compiled UNMODIFIED against this
    repository's include/ and library (`oracle/_ref/storygen_b200`), actually run on a 169M-shaped model
    with scripted stdin.

Both binaries are built by oracle/Makefile (`make ref-b200`) where /root/reference exists and travel to
the GPU box prebuilt; the tests skip when they are absent."""
import os
import subprocess
import time

import numpy as np
import pytest

from util import INCLUDE, ROOT, SEED_TOKEN, rel_err

pytestmark = pytest.mark.gpu

REF_DIR = os.path.join(ROOT, "oracle", "_ref")


def test_reference_header_runs_on_b200_hooks(pkg, make_model, tmp_path):
    from oracle.oracle import Oracle, read_ref_dump
    exe = os.path.join(REF_DIR, "ref_harness_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_harness_b200 not built (needs /root/reference at build time)")
    path = make_model(3, 768)
    orc = Oracle(path)
    toks, tok, refs = [], SEED_TOKEN, []
    for _ in range(8):
        toks.append(tok)
        lg = orc.forward(tok)
        refs.append(lg)
        tok = int(lg.argmax())
    tf = tmp_path / "toks.txt"
    tf.write_text("\n".join(map(str, toks)))
    dump = tmp_path / "hooks.bin"
    r = subprocess.run([exe, path, str(tf), str(dump)], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "loading: head_o" in r.stdout  # the reference's load UX (rwkv.cu:679)
    d = read_ref_dump(str(dump))
    assert d["steps"] == list(range(8))
    worst = max(rel_err(got, ref) for got, ref in zip(d["logits"], refs))
    print("reference rwkv.h on the B200 hooks vs oracle: worst logits rel err %.3g" % worst)
    assert worst < 1e-3
    for k in ("xy", "aa", "bb", "dd"):
        ref = orc.state[k]
        assert np.abs(d["state"][k] - ref).max() / max(np.abs(ref).max(), 1e-6) < 1e-3, k
    orc.close()


def test_storygen_runs_unmodified(pkg, make_model, tmp_path):
    """storygen.cpp looks for ../../../converter/model.bin and ../../../include/rwkv/tokenizer/vocab relative to its
    working directory (storygen.cpp:10,15) and loops forever; feed it one request and stop it after a while."""
    exe = os.path.join(REF_DIR, "storygen_b200")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/storygen_b200 not built (needs /root/reference at build time)")
    root = tmp_path / "tree"
    (root / "converter").mkdir(parents=True)
    os.symlink(make_model(12, 768), root / "converter" / "model.bin")
    os.symlink(INCLUDE, root / "include")
    cwd = root / "examples" / "storygen" / "build"
    cwd.mkdir(parents=True)
    p = subprocess.Popen([exe], cwd=str(cwd), stdin=subprocess.PIPE, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    p.stdin.write(b"a tale of two GPUs\n")
    p.stdin.flush()
    deadline = time.time() + 90
    out = b""
    os.set_blocking(p.stdout.fileno(), False)
    marker = b"Describe the story you want written:>"
    while time.time() < deadline:
        chunk = p.stdout.read()
        if chunk:
            out += chunk
        if marker in out and len(out.split(marker, 1)[1]) > 200:
            break  # well over 16 generated tokens after the request
        if p.poll() is not None:
            break
        time.sleep(0.2)
    p.kill()
    p.wait()
    text = out.decode(errors="replace")
    assert "Loaded model" in text, text[-2000:]
    assert marker.decode() in text, text[-2000:]
    generated = text.split(marker.decode(), 1)[1]
    print("storygen generated %d characters after the request" % len(generated))
    assert len(generated) > 200, text[-2000:]
