"""Build and run stream_probe.cu (the token kernel's weight-stream geometry: attainable HBM read rate and exchange-load
latency per bytes in flight and bulk-copy size) on GPU 0, after the card's name, power limit and top SM clock.
usage: python stream_probe.py [GiB per setting, default 4]"""
import os
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import build  # noqa: E402

subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], check=False)
with tempfile.TemporaryDirectory() as td:
    exe = os.path.join(td, "stream_probe")
    subprocess.run([build.nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-o", exe,
                    os.path.join(HERE, "stream_probe.cu")], check=True)
    sys.exit(subprocess.run([exe] + sys.argv[1:2]).returncode)
