#!/usr/bin/env python
"""Pinned host -> device copy bandwidth by size and number of streams (what bounds the upload leg of the e2e step)."""
import numpy as np, torch
import harness
def t(fn, n=10): return float(np.mean(harness.wall_ms(fn, n, warmup=1)[0]))
print(", ".join(harness.card().values()))
for mb in (8, 40, 200):
    h = torch.empty(mb*1024*1024//4, dtype=torch.float32).pin_memory(); d = torch.empty_like(h, device="cuda")
    ms = t(lambda: d.copy_(h, non_blocking=True)); print(f"{mb:4d} MB single copy: {ms:6.2f} ms = {mb/1024/ms*1e3:6.1f} GB/s")
    for k in (2, 4):
        streams = [torch.cuda.Stream() for _ in range(k)]
        hs = h.chunk(k); ds = d.chunk(k)
        def split():
            cur = torch.cuda.current_stream()
            for s_, a, b in zip(streams, hs, ds):
                s_.wait_stream(cur)
                with torch.cuda.stream(s_): b.copy_(a, non_blocking=True)
            for s_ in streams: cur.wait_stream(s_)
        ms = t(split); print(f"{mb:4d} MB on {k} streams: {ms:6.2f} ms = {mb/1024/ms*1e3:6.1f} GB/s")
x = torch.empty((5, 10, 1_000_000), dtype=torch.float32).pin_memory(); dx = torch.empty((10, 1_000_000), device="cuda")
print("view is_pinned:", x[3].is_pinned(), " 40 MB view copy:", t(lambda: dx.copy_(x[3], non_blocking=True)), "ms")
