"""Tensor-parallel checkpoint loading on one GPU: a safetensors file shaped like transformer layers in bf16 (per layer q, k, v, o
[h, h], gate and up [4h, h], down [h, 4h], two 1-D norms; h = 4096) is written into a pinned-once mem arena in 4 MiB blocks, then
rank 0's share of it is loaded these ways:
  whole           safetensors.load_file of every tensor (what one GPU holding the whole model does)
  strided_w{2,8}  load_file(slices=...) of rank 0's tensor-parallel slices at world 2 and 8: column-parallel tensors (q, k, v, gate,
                  up) on dim 0, row-parallel ones (o, down) on dim 1, norms whole -- one strided range per tensor
  per_row_w{2,8}  the same bytes through Reader.readv_device, one plain range per row of every dim-1 slice
For each leg: seconds (median of --steps after one warm-up step; allocation, the read and the CRC verification result included), GB/s
over the bytes the plan fetches and over the bytes delivered, the span count of the plan, the host time spent building the ranges and
planning them (timed separately), and the peak HBM allocated during the leg.  Prints one JSON line with the card's name and power limit.

    python tools/tp_load_bench.py [--gib 16] [--steps 3]
"""
import argparse
import json
import os
import shutil
import struct
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.readv_bench import card  # noqa: E402

BLOCK = 4 << 20
MIB = 1 << 20
COLUMN = ("q", "k", "v", "gate", "up")  # split on dim 0 (output features)
ROW = ("o", "down")                     # split on dim 1 (input features)


def layer_shapes(h):
    return [("q", (h, h)), ("k", (h, h)), ("v", (h, h)), ("o", (h, h)), ("gate", (4 * h, h)), ("up", (4 * h, h)), ("down", (h, 4 * h)),
            ("in_norm", (h,)), ("post_norm", (h,))]


def header_for(n_layers, h):
    hd, off, shapes = {}, 0, {}
    for l in range(n_layers):
        for kind, shape in layer_shapes(h):
            name = "layers.%d.%s" % (l, kind)
            nbytes = 2
            for x in shape:
                nbytes *= x
            hd[name] = {"dtype": "BF16", "shape": list(shape), "data_offsets": [off, off + nbytes]}
            shapes[name] = (kind, shape)
            off += nbytes
    hd["__metadata__"] = {"format": "pt"}
    raw = json.dumps(hd).encode()
    raw += b" " * (-(8 + len(raw)) % 8)
    return struct.pack("<Q", len(raw)) + raw, off, shapes


def rank_slices(shapes, world, rank=0):
    out = {}
    for name, (kind, shape) in shapes.items():
        dim = 0 if kind in COLUMN else 1 if kind in ROW else None
        if dim is not None:
            out[name] = (dim, rank * shape[dim] // world, (rank + 1) * shape[dim] // world)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16.0)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--dir", default="")
    args = ap.parse_args()

    import numpy as np
    import torch
    from curvine_b200 import fs as F
    from curvine_b200 import safetensors as ST

    assert torch.cuda.is_available(), "tp_load_bench needs a CUDA device"
    torch.cuda.set_device(0)
    h = args.hidden
    n_layers = max(1, int(args.gib * (1 << 30)) // (32 * h * h))
    head, data_len, shapes = header_for(n_layers, h)
    n = len(head) + data_len
    path = "/tp.safetensors"
    d = tempfile.mkdtemp(prefix="cvtpb", dir=args.dir or ("/dev/shm" if os.path.isdir("/dev/shm") else None))
    seg = 256 * MIB
    cap = (n + BLOCK + seg - 1) // seg * seg + seg
    w = F.MiniWorker(["[MEM:%d]%s/arena" % (cap, d)], extra_worker='mem_arena = true\narena_segment = "%d"\narena_reuse_delay = "0ms"\n' % seg)
    try:
        t0 = time.time()
        rng = np.random.default_rng(1)
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
            wr = wfs.create(path, 4343, BLOCK, w.port, chunk_size=1 << 20)
            wr.write(head)
            pat = rng.integers(0, 256, size=64 * MIB + 4096, dtype=np.uint8).tobytes()
            left, k = data_len, 0
            while left:
                step = min(left, 64 * MIB)
                wr.write(pat[k % 4096:k % 4096 + step])
                left -= step
                k += 1
            man = wr.complete()
        write_sec = time.time() - t0
        b200 = ('fetch_threads = 16\nverify_batch = 16\ncopy_group = 8\ngpu_chunk_size = "4MB"\nzero_copy = true\nregister_threads = 16\n'
                'arena_register_slice = "256MB"\narena_preregister = ["%s/arena"]\n' % d)
        start, ents = ST.parse_header(lambda o, k: head[o:o + k], n)
        with F.CurvineFileSystem(F.client_conf(short_circuit=True, b200=b200)) as fs:
            fs.load_namespace(man)
            fs.preregister()
            fs.wait_registered()
            st = torch.cuda.current_stream()

            def strided_ranges(slices):
                plan = ST.plan_ranges(start, ents, list(ents), slices)
                return [(r[0], r[1], r[2], r[3], 0, r[4]) for _, _, _, r in plan if r is not None]

            def per_row_ranges(slices, ptrs=None):
                """one plain range per row of every slice; ptrs (name -> data_ptr) places them, else 0"""
                out = []
                for name, (dt, shape, b, e) in ents.items():
                    p = ptrs[name] if ptrs else 0
                    if name not in slices:
                        out.append((start + b, e - b, p))
                        continue
                    dim, s0, s1 = slices[name]
                    if dim == 0:
                        inner = 2 * shape[1]
                        out.append((start + b + s0 * inner, (s1 - s0) * inner, p))
                        continue
                    row_len, pitch = (s1 - s0) * 2, shape[1] * 2
                    f0 = start + b + s0 * 2
                    out.extend((f0 + k * pitch, row_len, p + k * row_len if ptrs else 0) for k in range(shape[0]))
                return out

            def load_per_row(slices):
                out = {}
                for name, (dt, shape, _, _) in ents.items():
                    sh = list(shape)
                    if name in slices:
                        dim, s0, s1 = slices[name]
                        sh[dim] = s1 - s0
                    out[name] = torch.empty(sh, dtype=dt, device="cuda")
                with fs.open(path) as r:
                    r.readv_device(per_row_ranges(slices, {k: t.data_ptr() for k, t in out.items()}), st.cuda_stream)
                    assert r.verify()[1] == 0
                return out

            legs = {"whole": (lambda: ST.load_file(fs, path), {}, "strided")}
            for world in (2, 8):
                sl = rank_slices(shapes, world)
                legs["strided_w%d" % world] = ((lambda s=sl: ST.load_file(fs, path, slices=s)), sl, "strided")
                legs["per_row_w%d" % world] = ((lambda s=sl: load_per_row(s)), sl, "per_row")
            res = {k: [] for k in legs}
            peak = {k: 0 for k in legs}
            for step in range(args.steps + 1):  # step 0 warms every leg up; legs alternate within a step
                for k, (fn, _, _) in legs.items():
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    t = time.perf_counter()
                    out = fn()
                    st.synchronize()
                    sec = time.perf_counter() - t
                    peak[k] = max(peak[k], torch.cuda.max_memory_allocated() - base)
                    del out
                    if step:
                        res[k].append(sec)
            info = {}
            with fs.open(path) as r:
                for k, (_, sl, form) in legs.items():
                    t = time.perf_counter()
                    if form == "strided":
                        rs = strided_ranges(sl)
                        spans, nblocks, fetch = r.readv_strided_plan(rs)
                        delivered = sum(x[1] * x[2] for x in rs)
                    else:
                        rs = per_row_ranges(sl)
                        spans, nblocks, fetch = r.readv_plan(rs)
                        delivered = sum(x[1] for x in rs)
                    host = time.perf_counter() - t
                    med = sorted(res[k])[len(res[k]) // 2]
                    info[k] = {"sec": [round(x, 4) for x in res[k]], "sec_median": round(med, 4), "ranges": len(rs), "spans": len(spans),
                               "touched_blocks": nblocks, "fetched_bytes": fetch, "delivered_bytes": delivered,
                               "GBps_fetched": round(fetch / med / 1e9, 2), "GBps_delivered": round(delivered / med / 1e9, 2),
                               "host_ranges_and_plan_sec": round(host, 4), "peak_hbm_bytes": peak[k]}
        name, power = card()
        print(json.dumps({"card": name, "power_limit": power, "file_bytes": n, "layers": n_layers, "hidden": h, "block_bytes": BLOCK,
                          "steps": args.steps, "write_sec": round(write_sec, 2), "legs": info}))
    finally:
        w.stop()
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
