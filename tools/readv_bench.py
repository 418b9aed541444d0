"""Checkpoint loading on one GPU: a safetensors file shaped like a model checkpoint (about 300 tensors, 4 KiB biases next to matrices of
up to 500 MiB, so most tensor edges fall inside 4 MiB blocks) is written into a pinned-once mem arena, then timed three ways with CUDA
events on the calling stream:
  (a) read_to_tensor of the whole file (one flat uint8 buffer: the baseline)
  (b) safetensors.load_file of every tensor (one vectored read into ~300 separate tensors)
  (c) safetensors.load_file of every other tensor
Each time includes allocation and the CRC verification result.  For (c) the plan's fetched-byte count is printed beside the selected bytes
and the bound "selected + two blocks per selected tensor", so what the read moves can be checked without a profiler.  Prints one JSON
line with the card's name and power limit.

    python tools/readv_bench.py [--gib 16] [--tensors 300] [--steps 3]
"""
import argparse
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

BLOCK = 4 << 20
MIB = 1 << 20


def tensor_sizes(rng, n_tensors, total):
    import numpy as np
    """Half small (4-64 KiB) and half large tensors in random order, large ones capped at 500 MiB, summing to about `total` bytes; even
    sizes (BF16)."""
    n_small = n_tensors // 2
    small = [int(x) & ~1 for x in rng.integers(4096, 65536, size=n_small)]
    w = np.exp(rng.uniform(0.0, np.log(60.0), size=n_tensors - n_small))
    big = [min(500 * MIB, int(x)) & ~1 for x in w / w.sum() * (total - sum(small))]
    both = big + small
    return [both[i] for i in rng.permutation(n_tensors)]


def header_for(sizes):
    h, off = {}, 0
    for i, s in enumerate(sizes):
        h["t%03d" % i] = {"dtype": "BF16", "shape": [s // 2], "data_offsets": [off, off + s]}
        off += s
    h["__metadata__"] = {"format": "pt"}
    raw = json.dumps(h).encode()
    raw += b" " * (-(8 + len(raw)) % 8)
    return struct.pack("<Q", len(raw)) + raw, off


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], stdout=subprocess.PIPE,
                             stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip()
        name, power = [x.strip() for x in out.split(",")[:2]]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=16.0)
    ap.add_argument("--tensors", type=int, default=300)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--dir", default="")
    args = ap.parse_args()

    import numpy as np
    import torch
    from curvine_b200 import fs as F
    from curvine_b200 import safetensors as ST

    assert torch.cuda.is_available(), "readv_bench needs a CUDA device"
    torch.cuda.set_device(0)
    rng = np.random.default_rng(1)
    sizes = tensor_sizes(rng, args.tensors, int(args.gib * (1 << 30)))
    head, data_len = header_for(sizes)
    n = len(head) + data_len
    d = tempfile.mkdtemp(prefix="cvrvb", dir=args.dir or ("/dev/shm" if os.path.isdir("/dev/shm") else None))
    seg = 256 * MIB
    cap = (n + BLOCK + seg - 1) // seg * seg + seg
    w = F.MiniWorker(["[MEM:%d]%s/arena" % (cap, d)], extra_worker='mem_arena = true\narena_segment = "%d"\narena_reuse_delay = "0ms"\n' % seg)
    try:
        # the file goes through the worker (writes into the arena are not short-circuit), 64 MiB at a time from one random buffer
        t0 = time.time()
        with F.CurvineFileSystem(F.client_conf(short_circuit=False)) as wfs:
            wr = wfs.create("/ckpt.safetensors", 4242, BLOCK, w.port, chunk_size=1 << 20)
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
        with F.CurvineFileSystem(F.client_conf(short_circuit=True, b200=b200)) as fs:
            fs.load_namespace(man)
            fs.preregister()
            fs.wait_registered()
            st = torch.cuda.current_stream()

            def timed(fn):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(st)
                out = fn()
                e1.record(st)
                e1.synchronize()
                return e0.elapsed_time(e1) / 1e3, out

            names = list(ST.parse_header(lambda o, k: head[o:o + k], n)[1])
            half = names[::2]
            legs = {"a_read_to_tensor": lambda: fs.read_to_tensor("/ckpt.safetensors"),
                    "b_load_file_all": lambda: ST.load_file(fs, "/ckpt.safetensors"),
                    "c_load_file_every_other": lambda: ST.load_file(fs, "/ckpt.safetensors", names=half)}
            res = {k: [] for k in legs}
            for step in range(args.steps + 1):  # step 0 warms every leg up; legs alternate within a step
                for k, fn in legs.items():
                    sec, out = timed(fn)
                    del out
                    if step:
                        res[k].append(sec)
            start, ents = ST.parse_header(lambda o, k: head[o:o + k], n)
            with fs.open("/ckpt.safetensors") as r:
                ranges = [(start + ents[k][2], ents[k][3] - ents[k][2], 0) for k in half]
                spans, nblocks, fetch = r.readv_plan(ranges)
                direct = sum(1 for s in spans if s[4])
            sel = sum(x[1] for x in ranges)
        name, power = card()
        med = {k: sorted(v)[len(v) // 2] for k, v in res.items()}
        out = {"card": name, "power_limit": power, "file_bytes": n, "tensors": len(sizes), "block_bytes": BLOCK, "steps": args.steps,
               "write_sec": round(write_sec, 2),
               "sec": {k: [round(x, 4) for x in v] for k, v in res.items()},
               "GBps_median": {"a_read_to_tensor": n / med["a_read_to_tensor"] / 1e9, "b_load_file_all": data_len / med["b_load_file_all"] / 1e9,
                               "c_load_file_every_other": sel / med["c_load_file_every_other"] / 1e9},
               "b_rate_over_a_rate": (data_len / med["b_load_file_all"]) / (n / med["a_read_to_tensor"]),
               "c_plan": {"selected_bytes": sel, "fetched_bytes": fetch, "bound_selected_plus_two_blocks_each": sel + 2 * BLOCK * len(half),
                          "touched_blocks": nblocks, "direct_spans": direct, "spans": len(spans)}}
        print(json.dumps(out))
    finally:
        w.stop()
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
