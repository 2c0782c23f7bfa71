"""A/B the replayed denoising step under several environment settings in ONE GPU call: each configuration runs
tools/step_timing.py in its own process (the library reads its knobs once) for every batch size; prints one table.

    python tools/ab_step.py "base:" "fold:IMAGD_FOLD_LN=1" "bulk:IMAGD_GEMM_BULK_STORE=1" [--batches 1,8]
"""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
args = [a for a in sys.argv[1:] if not a.startswith("--")]
batches = [1, 8]
for a in sys.argv[1:]:
    if a.startswith("--batches"):
        batches = [int(v) for v in a.split("=", 1)[1].split(",")] if "=" in a else batches
configs = []
for a in args or ["base:"]:
    name, _, envs = a.partition(":")
    configs.append((name, dict(kv.split("=", 1) for kv in envs.split(",") if kv)))
rows = []
for name, env in configs:
    for B in batches:
        e = dict(os.environ, B=str(B), **env)
        out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "step_timing.py")], env=e, capture_output=True,
                             text=True, timeout=600)
        m = re.search(r"graph-replayed step ([0-9.]+) ms \((\d+) kernels\).*full image ([0-9.]+) ms", out.stdout)
        rows.append((name, B, m.groups() if m else ("FAILED", "-", (out.stderr or out.stdout)[-300:])))
        print(f"{name:12s} B={B:<3d} " + (f"step {m.group(1)} ms, {m.group(2)} kernels, image {m.group(3)} ms" if m
                                        else f"FAILED: {(out.stderr or out.stdout)[-300:]}"), flush=True)
