"""Config C4 (model distribution): a checkpoint file, mem tier, every GPU ends up holding ALL bytes in file order.

  torchrun --nproc-per-node G tools/c4_allgather.py --gib 32

Every GPU holds the whole file twice over (the file-order result and the all-gather staging buffer) plus its shard, so 32 GiB
is the largest power of two that fits an 80 GB H100.

Each rank ingests its round-robin shard (cv_read_device_sharded, CRC-32C verified on the GPU), then the exchange runs two ways:
  A  NCCL all_gather_into_tensor (in place) + cvk_deinterleave_blocks            (collective, then a 2N HBM pass)
  B  cvk_gather_shards_p2p: ONE kernel pulls every block straight from its owner's HBM over NVLink (peer pointers from
     torch symmetric memory) into file order -- no gathered staging buffer, no second pass
and every GPU re-verifies the whole file with K1 against the manifest.  Times are CUDA events, max over ranks."""
import argparse
import ctypes
import json
import os
import shutil
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
BLOCK = 4 << 20


def main_bench(args, emit):
    """bench.py --config c4: the same measurement, printed as ONE line in the bench contract (rank 0)."""
    a = argparse.Namespace(gib=32.0 if args.gib_per_gpu == 16.0 else args.gib_per_gpu * args.gpus, skip_nccl=False, arena=args.tier == "arena", emit=emit)
    return run(a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=32.0)
    ap.add_argument("--skip-nccl", action="store_true")
    ap.add_argument("--arena", type=int, default=1, help="mem tier = pinned-once arenas (one per GPU) instead of one tmpfs file per block")
    a = ap.parse_args()
    a.emit = None
    return run(a)


def run(a):
    import numpy as np
    import torch
    import torch.distributed as dist
    from curvine_b200 import _lib, fs as F, kernels as K
    rank, world, local = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    if world == 1:  # a single-rank "group" keeps the code below uniform (no exchange happens)
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29517")
        dist.init_process_group("nccl", rank=0, world_size=1, device_id=torch.device("cuda", local))
    else:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    L = _lib.lib()
    os.dup2(2, 1) if rank != 0 else None
    n = int(a.gib * (1 << 30)) // BLOCK * BLOCK
    nb = n // BLOCK
    per = (nb + world - 1) // world
    payload = [None, None]
    d = None
    if rank == 0:
        d = tempfile.mkdtemp(prefix="cvc4_", dir="/dev/shm")
        if a.arena:
            cap = per * BLOCK + (1 << 30) + (64 << 20)
            w = F.MiniWorker(["[MEM:%d]%s/a%d" % (cap, d, g) for g in range(world)], hostname="localhost",
                             extra_worker='mem_arena = true\narena_segment = "1GB"\narena_numa = [%s]\n' % ", ".join(str(int(L.cv_gpu_numa_node(g))) for g in range(world)))
        else:
            w = F.MiniWorker(["[MEM]" + d], hostname="localhost")
        L.cv_synth_set_shard_world(world)
        man = w.create_file("/ckpt", 777, n, BLOCK, threads=64)
        payload = [man, d]
    dist.broadcast_object_list(payload, src=0)
    man, d = payload[0], payload[1]
    exp = np.zeros(nb, dtype=np.uint32)
    for line in man.splitlines():
        if line.startswith("block "):
            f = line.split()
            exp[int(f[1]) & 0xFFFFFF] = int(f[5], 16)
    res = {"world": world, "file_bytes": n, "blocks": nb}
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def maxr(x):
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    try:
        conf = F.client_conf(hostname="localhost", short_circuit=True,
                             b200='device = %d\nfetch_threads = 8\nzero_copy = true\nregister_cache = "%dGB"\ncopy_group = 8\nverify_batch = 16\n'
                                  'arena_preregister = ["%s/a%d"]\n' % (local, int(a.gib / world * 1.5) + 2, d, rank))
        fs = F.CurvineFileSystem(conf)
        fs.load_namespace(man)
        t0 = time.time()
        fs.preregister()
        fs.wait_registered()
        res["mount_ms"] = (time.time() - t0) * 1e3
        final = torch.empty(n, dtype=torch.uint8, device="cuda")
        # the shard lives in symmetric memory: every rank gets a directly loadable pointer to every peer's shard
        if world > 1:
            import torch.distributed._symmetric_memory as symm_mem
            shard = symm_mem.empty(per * BLOCK, dtype=torch.uint8, device="cuda")
            hdl = symm_mem.rendezvous(shard, dist.group.WORLD.group_name)
            peers = [int(p) for p in hdl.buffer_ptrs]
        else:
            shard = torch.empty(per * BLOCK, dtype=torch.uint8, device="cuda")
            peers = [int(shard.data_ptr())]
        stream = torch.cuda.current_stream().cuda_stream
        # ---- ingest (twice; with the arena tier the first pass is already DMA out of pinned segments)
        for rep in range(2):
            torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
            e0, e1 = ev(), ev()
            e0.record()
            r = fs.open("/ckpt")
            got = r.read_device_sharded(rank, world, shard.data_ptr(), per * BLOCK, stream)
            s, bad, ver = r.verify()
            e1.record(); e1.synchronize()
            r.complete()
            assert bad == 0 and ver == len(range(rank, nb, world))
            res["ingest_ms_rep%d" % rep] = maxr(e0.elapsed_time(e1))
        res["ingest_GBps"] = n / res["ingest_ms_rep1"] / 1e6
        res["ingest_first_read_GBps"] = n / res["ingest_ms_rep0"] / 1e6
        # ---- full-file verify helper (K1 over the final buffer on every GPU)
        d_off = torch.arange(nb, dtype=torch.int64, device="cuda") * BLOCK
        d_len = torch.full((nb,), BLOCK, dtype=torch.int64, device="cuda")
        d_exp = torch.from_numpy(exp.view(np.int32)).cuda()
        d_crc = torch.empty(nb, dtype=torch.int32, device="cuda")

        def verify_final(tag):
            d_bad = torch.zeros(1, dtype=torch.int32, device="cuda")
            e0, e1 = ev(), ev()
            e0.record()
            K.crc_blocks_raw(final.data_ptr(), d_off, d_len, nb, 1, n, d_crc)
            K.verify_crcs(d_crc, d_exp, d_bad)
            e1.record(); e1.synchronize()
            assert int(d_bad.item()) == 0, "%s: %d bad blocks" % (tag, int(d_bad.item()))
            res[tag + "_verify_ms"] = maxr(e0.elapsed_time(e1))

        # ---- B: fused peer gather over NVLink
        for rep in range(3):
            final.zero_()
            torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
            e0, e1 = ev(), ev()
            e0.record()
            K.gather_shards_p2p(peers, BLOCK, nb, n, final)
            e1.record(); e1.synchronize()
            res["p2p_gather_ms_rep%d" % rep] = maxr(e0.elapsed_time(e1))
        verify_final("p2p")
        torch.cuda.synchronize(); dist.barrier()
        res["p2p_gather_GBps_into_each_gpu"] = n / res["p2p_gather_ms_rep2"] / 1e6
        res["p2p_nvlink_GBps_per_gpu"] = n * (world - 1) / world / res["p2p_gather_ms_rep2"] / 1e6
        # ---- A: NCCL all-gather + de-interleave
        if not a.skip_nccl:
            gathered = torch.empty(world * per * BLOCK, dtype=torch.uint8, device="cuda")
            mine = gathered[rank * per * BLOCK:(rank + 1) * per * BLOCK]
            mine.copy_(shard)
            for rep in range(2):
                final.zero_()
                torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
                e0, e1, e2 = ev(), ev(), ev()
                e0.record()
                dist.all_gather_into_tensor(gathered, mine)
                e1.record()
                K.deinterleave_blocks(gathered, per * BLOCK, world, BLOCK, nb, n, final)
                e2.record(); e2.synchronize()
                res["nccl_allgather_ms_rep%d" % rep] = maxr(e0.elapsed_time(e1))
                res["deinterleave_ms_rep%d" % rep] = maxr(e1.elapsed_time(e2))
            verify_final("nccl")
            res["nccl_total_ms"] = res["nccl_allgather_ms_rep1"] + res["deinterleave_ms_rep1"]
        fs.close()
    finally:
        torch.cuda.synchronize()
        dist.barrier()
        if rank == 0:
            w.stop()
            shutil.rmtree(d, ignore_errors=True)
    dist.destroy_process_group()
    if rank != 0:
        return
    if a.emit is None:
        sys.stdout.write(json.dumps(res) + "\n")
        return
    # the bench contract line: value = file bytes / (first-read ingest + the faster exchange), per GPU every byte of the file
    exch = min(res["p2p_gather_ms_rep2"], res.get("nccl_total_ms", 1e30))
    total_ms = res["ingest_ms_rep0"] + exch
    a.emit({"metric": "model distribution: checkpoint GB/s into EVERY GPU's HBM in file order (CRC-verified)", "value": n / total_ms / 1e6, "unit": "GB/s",
            "n_gpus": world, "steps": 1, "warmup": 0, "ms_per_step": total_ms, "higher_is_better": True, "scaling": "strong", "vs_baseline": None,
            "dtype": "u8", "data": "synthetic",
            "config": {"workload": "C4: %.1f GiB checkpoint, 4 MiB blocks, mem tier (%s), every GPU ingests its round-robin shard then pulls the rest from its peers"
                                   % (n / 2 ** 30, "arena" if a.arena else "files"), "file_bytes": n, "block_bytes": BLOCK},
            "ingest": {"first_read_ms": res["ingest_ms_rep0"], "first_read_GBps": n / res["ingest_ms_rep0"] / 1e6, "reread_ms": res["ingest_ms_rep1"], "mount_ms": res.get("mount_ms")},
            "exchange_p2p_fused": {"ms": res["p2p_gather_ms_rep2"], "GBps_into_each_gpu": res["p2p_gather_GBps_into_each_gpu"],
                                   "nvlink_GBps_per_gpu": res["p2p_nvlink_GBps_per_gpu"], "frac_of_nvlink4_450GBps": res["p2p_nvlink_GBps_per_gpu"] / 450.0,
                                   "what": "cvk_gather_shards_p2p: one K3-bodied kernel per GPU reads every block out of its owner's HBM (peer pointers, symmetric memory) into file order"},
            "exchange_nccl": {"allgather_ms": res.get("nccl_allgather_ms_rep1"), "deinterleave_ms": res.get("deinterleave_ms_rep1"), "total_ms": res.get("nccl_total_ms"),
                              "what": "all_gather_into_tensor + cvk_deinterleave_blocks"},
            "verify_ms": {"p2p": res.get("p2p_verify_ms"), "nccl": res.get("nccl_verify_ms")},
            # the step is end to end by construction: the checkpoint starts in the worker's host memory and ends, verified, in every GPU's HBM
            "e2e": {"value": n / total_ms / 1e6, "unit": "GB/s", "h2d_bytes_per_step": n, "d2h_bytes_per_step": 4 * ((n + BLOCK - 1) // BLOCK + 4 * world),
                    "what": "cv_read_device_sharded on every rank (host memory -> HBM, CRC-verified) + the exchange that leaves the whole file on every GPU"},
            "gpu_launches": int(K.launch_count()), "raw": res})


if __name__ == "__main__":
    main()
