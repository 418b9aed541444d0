"""Cast on load on one GPU: a float32 safetensors file shaped like transformer layers (per layer q, k, v, o [h, h], gate and up [4h, h],
down [h, 4h], two 1-D norms; h = 4096) is written into a pinned-once mem arena in 4 MiB blocks, then loaded these ways:
  f32            safetensors.load_file as stored
  f32_then_to    load_file, then .to(torch.bfloat16) tensor by tensor, each float32 tensor freed as soon as its copy exists
  cast_bf16      load_file(dtype=torch.bfloat16): converted on the GPU out of the verified staging, in the same read
  cast_bf16_w8   load_file(slices=..., dtype=torch.bfloat16) of rank 0 of world 8 (column-parallel tensors on dim 0, row-parallel on dim 1)
For each leg: seconds (median of --steps after one warm-up step; allocation, the read and the CRC verification result included), GB/s
over the bytes the plan fetches, the bytes delivered, and the peak HBM torch allocated during the leg.  The reader's boundary staging
(at most 256 MiB, reused by every load) is allocated by the library, outside torch's allocator, and is not in those peaks.
A kernel leg times cvk_gather_cast alone on HBM-resident data (float32 -> bfloat16 and bfloat16 -> float32 over 1 GiB of source, CUDA
events, after warm-up) and reports (source + destination bytes) / time.  Prints one JSON line with the card's name and power limit.

    python tools/cast_load_bench.py [--gib 16] [--steps 3]
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
from tools.tp_load_bench import layer_shapes, rank_slices  # noqa: E402

BLOCK = 4 << 20
MIB = 1 << 20
HBM_PEAK_TBPS = 3.35  # H100 SXM data sheet


def header_for(n_layers, h):
    hd, off, shapes = {}, 0, {}
    for l in range(n_layers):
        for kind, shape in layer_shapes(h):
            name = "layers.%d.%s" % (l, kind)
            nbytes = 4
            for x in shape:
                nbytes *= x
            hd[name] = {"dtype": "F32", "shape": list(shape), "data_offsets": [off, off + nbytes]}
            shapes[name] = (kind, shape)
            off += nbytes
    hd["__metadata__"] = {"format": "pt"}
    raw = json.dumps(hd).encode()
    raw += b" " * (-(8 + len(raw)) % 8)
    return struct.pack("<Q", len(raw)) + raw, off, shapes


def kernel_leg(torch, reps=10):
    """cvk_gather_cast over 1 GiB of HBM-resident source, one segment of one row: -> {conversion: numbers}"""
    from curvine_b200 import _lib
    from curvine_b200 import kernels as K
    out = {}
    for name, sdt, ddt in (("f32_to_bf16", torch.float32, torch.bfloat16), ("bf16_to_f32", torch.bfloat16, torch.float32)):
        n = (1 << 30) // sdt.itemsize
        src = torch.randn(n, device="cuda").to(sdt)
        dst = torch.empty(n, dtype=ddt, device="cuda")
        code = {torch.float32: _lib.DTYPE_F32, torch.bfloat16: _lib.DTYPE_BF16}
        segs, total = K.cast_segs_to_device([(0, 0, n, 1, 0, 0, code[sdt], code[ddt])], "cuda")
        for _ in range(3):
            K.gather_cast(src, segs, 1, total, dst)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(reps):
            a.record()
            K.gather_cast(src, segs, 1, total, dst)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        assert torch.equal(dst[:1 << 20].view(torch.int16 if ddt.itemsize == 2 else torch.int32),
                           src[:1 << 20].cpu().to(ddt).cuda().view(torch.int16 if ddt.itemsize == 2 else torch.int32)) or bool(
            torch.isnan(src[:1 << 20].float()).any())
        med = sorted(ms)[len(ms) // 2]
        moved = n * (sdt.itemsize + ddt.itemsize)
        out[name] = {"source_bytes": n * sdt.itemsize, "ms": [round(x, 4) for x in ms], "ms_median": round(med, 4),
                     "TBps_src_plus_dst": round(moved / med / 1e9, 3), "fraction_of_3.35TBps": round(moved / med / 1e9 / HBM_PEAK_TBPS, 3)}
        del src, dst, segs
        torch.cuda.empty_cache()
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

    assert torch.cuda.is_available(), "cast_load_bench needs a CUDA device"
    torch.cuda.set_device(0)
    kern = kernel_leg(torch)
    h = args.hidden
    n_layers = max(1, int(args.gib * (1 << 30)) // (64 * h * h))
    head, data_len, shapes = header_for(n_layers, h)
    n = len(head) + data_len
    path = "/cast.safetensors"
    d = tempfile.mkdtemp(prefix="cvcab", dir=args.dir or ("/dev/shm" if os.path.isdir("/dev/shm") else None))
    seg = 256 * MIB
    cap = (n + BLOCK + seg - 1) // seg * seg + seg
    w = F.MiniWorker(["[MEM:%d]%s/arena" % (cap, d)], extra_worker='mem_arena = true\narena_segment = "%d"\narena_reuse_delay = "0ms"\n' % seg)
    try:
        t0 = time.time()
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
            wr = wfs.create(path, 4344, BLOCK, w.port, chunk_size=1 << 20)
            wr.write(head)
            # finite float32 values (a random bit pattern would make NaNs): normal values spread over many exponents
            pat = (np.random.default_rng(1).standard_normal(16 * MIB + 1024).astype(np.float32) * 1e3).tobytes()
            left, k = data_len, 0
            while left:
                step = min(left, 64 * MIB)
                o = 4 * (k % 1024)
                wr.write(pat[o:o + step])
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

            def then_to():
                out = ST.load_file(fs, path)
                for name in list(out):
                    out[name] = out[name].to(torch.bfloat16)  # the float32 tensor is freed here
                return out

            sl8 = rank_slices(shapes, 8)
            legs = {"f32": ((lambda: ST.load_file(fs, path)), {}, None),
                    "f32_then_to": (then_to, {}, None),
                    "cast_bf16": ((lambda: ST.load_file(fs, path, dtype=torch.bfloat16)), {}, torch.bfloat16),
                    "cast_bf16_w8": ((lambda: ST.load_file(fs, path, slices=sl8, dtype=torch.bfloat16)), sl8, torch.bfloat16)}
            res = {k: [] for k in legs}
            peak = {k: 0 for k in legs}
            delivered = {}
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
                    delivered[k] = sum(x.numel() * x.element_size() for x in out.values())
                    del out
                    if step:
                        res[k].append(sec)
            info = {}
            with fs.open(path) as r:
                for k, (_, sl, dt) in legs.items():
                    plan = ST.plan_ranges(start, ents, list(ents), sl, dt)
                    if dt is None:
                        _, nblocks, fetch = r.readv_strided_plan([(x[0], x[1], x[2], x[3], 0, x[4]) for _, _, _, x in plan if x is not None])
                    else:
                        _, nblocks, fetch = r.readv_cast_plan([(x[0], x[1], x[2], x[3], 0, x[4], x[5], x[6]) for _, _, _, x in plan if x is not None])
                    med = sorted(res[k])[len(res[k]) // 2]
                    info[k] = {"sec": [round(x, 4) for x in res[k]], "sec_median": round(med, 4), "touched_blocks": nblocks, "fetched_bytes": fetch,
                               "delivered_bytes": delivered[k], "GBps_fetched": round(fetch / med / 1e9, 2), "peak_hbm_bytes_torch": peak[k]}
        name, power = card()
        print(json.dumps({"card": name, "power_limit": power, "file_bytes": n, "layers": n_layers, "hidden": h, "block_bytes": BLOCK,
                          "steps": args.steps, "write_sec": round(write_sec, 2),
                          "note": "peaks are torch's allocator only; the reader's staging (<= 256 MiB) is allocated by the library",
                          "legs": info, "kernel": kern}))
    finally:
        w.stop()
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
