"""FP8 checkpoints on load on one GPU: a safetensors file shaped like transformer layers (per layer q, k, v, o [h, h], gate and up [4h, h],
down [h, 4h] as F8_E4M3, each with a float32 `<name>_scale_inv` of one scale per 128 x 128 tile, and two bfloat16 1-D norms; h = 4096)
is written into a pinned-once mem arena in 4 MiB blocks, then loaded these ways:
  torch_dequant   safetensors.load_file as stored, then on the GPU tensor by tensor (w.float() * s_full).to(torch.bfloat16), s_full the
                  scale grid expanded and cropped -- DeepSeek's formula; each FP8 weight and its float32 temporary freed as soon as done
  scaled_bf16     load_file(dtype=torch.bfloat16, scales=..., scale_block=(128, 128)): dequantized on the GPU out of the verified staging
  scaled_bf16_w8  the same with slices= of rank 0 of world 8 (column-parallel weights on dim 0, row-parallel on dim 1)
For each leg: seconds (median of --steps after one warm-up step; allocation, the reads and the CRC verification result included), GB/s
over the bytes the plans fetch (for the scaled legs both calls': the scales' read fetches every block holding a scale whole, and the
second call fetches those blocks again), the bytes delivered, and the peak HBM torch allocated during the leg.  The reader's boundary staging
(at most 256 MiB) is allocated by the library, outside torch's allocator, and is not in those peaks.
A kernel leg times cvk_gather_cast_scaled alone on HBM-resident data, F8_E4M3 -> bfloat16 over 1 GiB of source, with 128 x 128 float32
scales and without scales (CUDA events, after warm-up), and reports algorithmic bytes (source + destination + scales) / time.  Prints one
JSON line with the card's name and power limit.

    python tools/fp8_load_bench.py [--gib 4] [--steps 3]
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
TILE = 128
HBM_PEAK_TBPS = 3.35  # H100 SXM data sheet


def header_for(n_layers, h):
    """-> (header bytes, data length, {weight: (kind, shape)}, {weight: its scale}, [(name, dtype, nbytes)] in file order)"""
    hd, off, shapes, scales, order = {}, 0, {}, {}, []

    def add(name, dt, shape, size):
        nonlocal off
        n = size
        for x in shape:
            n *= x
        hd[name] = {"dtype": dt, "shape": list(shape), "data_offsets": [off, off + n]}
        order.append((name, dt, n))
        off += n

    for l in range(n_layers):
        for kind, shape in layer_shapes(h):
            name = "layers.%d.%s" % (l, kind)
            if len(shape) == 2:
                add(name, "F8_E4M3", shape, 1)
                add(name + "_scale_inv", "F32", (-(-shape[0] // TILE), -(-shape[1] // TILE)), 4)
                shapes[name], scales[name] = (kind, shape), name + "_scale_inv"
            else:
                add(name, "BF16", shape, 2)
    hd["__metadata__"] = {"format": "pt"}
    raw = json.dumps(hd).encode()
    raw += b" " * (-(8 + len(raw)) % 8)
    return struct.pack("<Q", len(raw)) + raw, off, shapes, scales, order


def dequant(torch, w, s, dtype):
    """DeepSeek's formula on the GPU: (w.float() * s_full).to(dtype)"""
    R, C = w.shape
    full = s.repeat_interleave(TILE, 0).repeat_interleave(TILE, 1)[:R, :C]
    return (w.float() * full).to(dtype)


def kernel_leg(torch, reps=10):
    """cvk_gather_cast_scaled over 1 GiB of HBM-resident F8_E4M3 source seen as [65536, 16384], one segment of one row, with and
    without 128 x 128 float32 scales -> {variant: numbers}"""
    from curvine_b200 import _lib
    from curvine_b200 import kernels as K
    R, C = 1 << 16, 1 << 14
    n = R * C
    src = torch.randint(0, 256, (n,), dtype=torch.uint8, device="cuda")
    src[(src & 0x7F) == 0x7F] = 0x3C  # no NaNs, so the check below can compare bits
    dst = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    s = torch.rand((R // TILE, C // TILE), device="cuda") * 2.0 ** -8
    segs, total = K.cast_segs_to_device([(0, 0, n, 1, 0, 0, _lib.DTYPE_F8_E4M3, _lib.DTYPE_BF16)], "cuda")
    out = {}
    for name, sc in (("scaled_f8e4m3_to_bf16", (s.data_ptr(), _lib.DTYPE_F32, TILE, TILE, C // TILE, C, 0, 0)), ("unscaled_f8e4m3_to_bf16", None)):
        d_sc = K.scale_segs_to_device([sc], "cuda")
        for _ in range(3):
            K.gather_cast_scaled(src, segs, d_sc, 1, total, dst)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(reps):
            a.record()
            K.gather_cast_scaled(src, segs, d_sc, 1, total, dst)
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        rows = 256  # the first 256 view rows against torch on the GPU
        w = src[:rows * C].view(torch.float8_e4m3fn).view(rows, C)
        want = dequant(torch, w, s[:rows // TILE], torch.bfloat16) if sc else w.to(torch.bfloat16)
        assert torch.equal(dst[:rows * C].view(torch.int16), want.reshape(-1).view(torch.int16)), name
        med = sorted(ms)[len(ms) // 2]
        moved = n + 2 * n + (s.numel() * 4 if sc else 0)
        out[name] = {"source_bytes": n, "ms": [round(x, 4) for x in ms], "ms_median": round(med, 4), "algorithmic_bytes": moved,
                     "TBps_algorithmic": round(moved / med / 1e9, 3), "fraction_of_3.35TBps": round(moved / med / 1e9 / HBM_PEAK_TBPS, 3)}
        del d_sc
    del src, dst, s, segs
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--dir", default="")
    args = ap.parse_args()

    import numpy as np
    import torch
    from curvine_b200 import fs as F
    from curvine_b200 import safetensors as ST

    assert torch.cuda.is_available(), "fp8_load_bench needs a CUDA device"
    torch.cuda.set_device(0)
    kern = kernel_leg(torch)
    h = args.hidden
    n_layers = max(1, int(args.gib * (1 << 30)) // (16 * h * h))
    head, data_len, shapes, scales, order = header_for(n_layers, h)
    n = len(head) + data_len
    path = "/fp8.safetensors"
    d = tempfile.mkdtemp(prefix="cvf8b", dir=args.dir or ("/dev/shm" if os.path.isdir("/dev/shm") else None))
    seg = 256 * MIB
    cap = (n + BLOCK + seg - 1) // seg * seg + seg
    w = F.MiniWorker(["[MEM:%d]%s/arena" % (cap, d)], extra_worker='mem_arena = true\narena_segment = "%d"\narena_reuse_delay = "0ms"\n' % seg)
    try:
        t0 = time.time()
        rng = np.random.default_rng(1)
        # E4M3 weights: every byte pattern but the two NaNs; scales 2^-12 .. 2^-4 as a checkpoint's scale_inv; norms near 1
        f8 = rng.integers(0, 256, size=16 * MIB + 1024, dtype=np.uint8)
        f8[(f8 & 0x7F) == 0x7F] = 0x3C
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
            wr = wfs.create(path, 4345, BLOCK, w.port, chunk_size=1 << 20)
            wr.write(head)
            k = 0
            for name, dt, nbytes in order:
                if dt == "F8_E4M3":
                    left = nbytes
                    while left:
                        step = min(left, 16 * MIB)
                        o = k % 1024
                        wr.write(f8[o:o + step].tobytes())
                        left -= step
                        k += 1
                elif dt == "F32":
                    wr.write(np.ldexp(rng.uniform(0.5, 1.0, nbytes // 4), rng.integers(-12, -3, nbytes // 4)).astype(np.float32).tobytes())
                else:
                    wr.write(torch.from_numpy(rng.uniform(0.5, 1.5, nbytes // 2).astype(np.float32)).to(torch.bfloat16).view(torch.int16).numpy().tobytes())
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

            def torch_dequant():
                out = ST.load_file(fs, path)
                for name, sname in scales.items():
                    out[name] = dequant(torch, out[name], out[sname], torch.bfloat16)  # the FP8 weight and the temporary are freed here
                return out

            sl8 = rank_slices(shapes, 8)
            bf = torch.bfloat16
            legs = {"torch_dequant": (torch_dequant, {}, None, None),
                    "scaled_bf16": ((lambda: ST.load_file(fs, path, dtype=bf, scales=scales, scale_block=(TILE, TILE))), {}, bf, scales),
                    "scaled_bf16_w8": ((lambda: ST.load_file(fs, path, slices=sl8, dtype=bf, scales=scales, scale_block=(TILE, TILE))), sl8, bf,
                                       scales)}
            res = {k: [] for k in legs}
            peak = {k: 0 for k in legs}
            delivered, check = {}, {}
            for step in range(args.steps + 1):  # step 0 warms every leg up; legs alternate within a step
                for k, (fn, _, _, _) in legs.items():
                    torch.cuda.synchronize()
                    base = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    t = time.perf_counter()
                    out = fn()
                    st.synchronize()
                    sec = time.perf_counter() - t
                    peak[k] = max(peak[k], torch.cuda.max_memory_allocated() - base)
                    delivered[k] = sum(x.numel() * x.element_size() for name, x in out.items() if not (k == "torch_dequant" and name.endswith("_scale_inv")))
                    if step == 0:  # the dequantized weights of layer 0 agree bit for bit between the legs
                        check[k] = {name: out[name].view(torch.int16).sum(dtype=torch.int64).item() for name in shapes if name.startswith("layers.0.")}
                    del out
                    if step:
                        res[k].append(sec)
            assert check["torch_dequant"] == check["scaled_bf16"], (check["torch_dequant"], check["scaled_bf16"])
            info = {}
            with fs.open(path) as r:
                for k, (_, sl, dt, scl) in legs.items():
                    plan = ST.plan_ranges(start, ents, list(ents), sl, dt, scl, (TILE, TILE) if scl else None)
                    if dt is None:
                        _, nblocks, fetch = r.readv_strided_plan([(x[0], x[1], x[2], x[3], 0, x[4]) for _, _, _, x in plan if x is not None])
                    else:  # the scaled read
                        _, nblocks, fetch = r.readv_cast_plan([(x[0], x[1], x[2], x[3], 0, x[4], x[5], x[6]) for _, _, _, x in plan if x is not None])
                    scale_fetch = 0
                    if scl:  # and the first call, which reads the scale tensors: it fetches (and verifies) every block holding a scale whole
                        used = dict.fromkeys(x[7][0] for _, _, _, x in plan if x is not None and x[7] is not None)
                        _, sblocks, scale_fetch = r.readv_strided_plan([(start + ents[n][2], ents[n][3] - ents[n][2], 1, 0, 0, 0) for n in used])
                        nblocks += sblocks
                    fetch += scale_fetch
                    med = sorted(res[k])[len(res[k]) // 2]
                    info[k] = {"sec": [round(x, 4) for x in res[k]], "sec_median": round(med, 4), "touched_blocks": nblocks, "fetched_bytes": fetch,
                               "fetched_bytes_scale_call": scale_fetch, "delivered_bytes": delivered[k], "GBps_fetched": round(fetch / med / 1e9, 2),
                               "peak_hbm_bytes_torch": peak[k]}
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
