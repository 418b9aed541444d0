"""TEST INFRASTRUCTURE ONLY: builds the product's host side AND its kernel source (curvine_b200/csrc/kernels.cu) for host cores:
the kernels run on the SIMT shim of this directory (simt_emu.h: a fiber per CUDA thread, real barrier / warp-collective
semantics), the runtime calls land on the host-memory stand-in of tests/mock_cuda.  The result is a library under /tmp with the
product's full C ABI (cv_* and cvk_*), which tests/test_kernels_on_simt_emu.py points the GPU parity tests at -- so the kernels'
algorithm is checked against the oracle on machines without a GPU as well.  The product library is built by curvine_b200/build.py
with nvcc; nothing under curvine_b200/ knows about this one.

kernels.cu is compiled from a mechanically rewritten copy (written to the build directory, never committed):
  * `kernel<<<grid, block, smem, stream>>>(args)`  ->  `cv_emu::cfg(grid, block, smem, stream)(kernel, args)`
  * `extern __shared__ T name[];`                   ->  `T* name = reinterpret_cast<T*>(cv_emu::dyn_smem());`
  * every inline-PTX statement                      ->  the cv_emu::ptx_* function that states what the instruction does
An instruction or construct the rewrite does not know stops the build: the shim has to be taught, not guess."""
import hashlib
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "curvine_b200", "csrc")
HOST = os.path.join(CSRC, "host")
MOCK = os.path.join(ROOT, "tests", "mock_cuda")


def _match_paren(s, i):
    """s[i] == '(' -> index of the matching ')', skipping string literals."""
    depth, j, n = 0, i, len(s)
    while j < n:
        c = s[j]
        if c == '"':
            j += 1
            while s[j] != '"':
                j += 2 if s[j] == "\\" else 1
        elif c == "(":
            depth += 1
        elif c == ")":
            depth -= 1
            if depth == 0:
                return j
        j += 1
    raise ValueError("unbalanced parenthesis")


def _split_top(s, sep):
    """split on `sep` outside (), {}, [], <> are NOT tracked (template commas are handled by the caller) and outside strings"""
    out, depth, cur, j = [], 0, "", 0
    while j < len(s):
        c = s[j]
        if c == '"':
            k = j + 1
            while s[k] != '"':
                k += 2 if s[k] == "\\" else 1
            cur += s[j:k + 1]
            j = k + 1
            continue
        if c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
        if c == sep and depth == 0:
            out.append(cur)
            cur = ""
        else:
            cur += c
        j += 1
    out.append(cur)
    return out


def _operands(section):
    """'"=r"(r.x), "l"(p)' -> ['r.x', 'p']"""
    out = []
    for item in _split_top(section, ","):
        item = item.strip()
        if not item:
            continue
        m = re.match(r'"[^"]*"\s*\((.*)\)\s*$', item, re.S)
        if not m:
            raise ValueError("asm operand not understood: %r" % item)
        out.append(m.group(1).strip())
    return out


def _ptx_call(text, ops):
    """one PTX statement + its operand expressions (asm order: outputs then inputs) -> C++"""
    t = " ".join(text.replace(";", " ").split())
    opcode = t.split(" ")[0]
    o = lambda k: "(" + ops[k] + ")"  # noqa: E731
    if re.fullmatch(r"ld\.global(\.nc)?(\.L1::no_allocate)?\.v4\.u32", opcode) and t.endswith("{%0,%1,%2,%3}, [%4]"):
        return "cv_emu::ptx_ld_v4(%s, %s, %s, %s, %s)" % (o(0), o(1), o(2), o(3), o(4))
    if opcode == "st.global.v4.u32" and t.endswith("[%0], {%1,%2,%3,%4}"):
        return "cv_emu::ptx_st_v4(%s, %s, %s, %s, %s)" % (o(0), o(1), o(2), o(3), o(4))
    if opcode == "ld.shared.v4.u32" and t.endswith("{%0,%1,%2,%3}, [%4]"):
        return "cv_emu::ptx_lds_v4(%s, %s, %s, %s, %s)" % (o(0), o(1), o(2), o(3), o(4))
    if opcode == "ld.shared.u32" and t.endswith("%0, [%1]"):
        return "cv_emu::ptx_lds_u32(%s, %s)" % (o(0), o(1))
    if opcode == "cp.async.cg.shared.global" and t.endswith("[%0], [%1], 16"):
        return "cv_emu::ptx_cp_async16(%s, %s)" % (o(0), o(1))
    if opcode == "cp.async.commit_group":
        return "cv_emu::ptx_cp_async_commit()"
    if opcode == "cp.async.wait_group" and t.endswith("%0"):
        return "cv_emu::ptx_cp_async_wait(%s)" % o(0)
    raise ValueError("PTX statement the SIMT shim does not know: %r" % text)


def rewrite(src):
    # 1. inline PTX
    out, i = "", 0
    for m in re.finditer(r"\basm\s*(volatile\s*)?\(", src):
        if m.start() < i:
            continue
        close = _match_paren(src, m.end() - 1)
        body = src[m.end():close]
        sections = []
        for part in _split_top(body, ":"):  # "::" (no outputs) yields an empty section
            sections.append(part.strip())
        strings = re.findall(r'"((?:[^"\\]|\\.)*)"', sections[0])
        ops = _operands(sections[1] if len(sections) > 1 else "") + _operands(sections[2] if len(sections) > 2 else "")
        out += src[i:m.start()] + _ptx_call("".join(strings), ops) + "\n" * src[m.start():close].count("\n")  # line numbers stay those of kernels.cu
        i = close + 1
    src = out + src[i:]
    # 2. dynamic shared memory
    src, n = re.subn(r"extern\s+__shared__\s+(\w+)\s+(\w+)\s*\[\s*\]\s*;", r"\1* \2 = reinterpret_cast<\1*>(cv_emu::dyn_smem());", src)
    # 3. launches
    out, i = "", 0
    while True:
        k = src.find("<<<", i)
        if k < 0:
            break
        # kernel expression: identifier, optionally followed by balanced template arguments, right before <<<
        j = k
        if src[j - 1] == ">":
            depth, j = 0, k - 1
            while True:
                if src[j] == ">":
                    depth += 1
                elif src[j] == "<":
                    depth -= 1
                    if depth == 0:
                        break
                j -= 1
        while j > 0 and (src[j - 1].isalnum() or src[j - 1] in "_:"):
            j -= 1
        kernel = src[j:k]
        e = src.find(">>>", k)
        conf = _split_top(src[k + 3:e], ",")
        if len(conf) != 4:
            raise ValueError("launch configuration with %d arguments: %r" % (len(conf), src[k:e + 3]))
        p = e + 3
        while src[p].isspace():
            p += 1
        if src[p] != "(":
            raise ValueError("launch without argument list: %r" % src[j:p + 10])
        out += src[i:j] + "cv_emu::cfg(%s)(%s, " % (", ".join(c.strip() for c in conf), kernel.strip())
        i = p + 1
    return out + src[i:]


def sources():
    host = [os.path.join(HOST, f) for f in sorted(os.listdir(HOST)) if f.endswith((".cc", ".cu")) and f != "gds.cc"]
    return host + [os.path.join(MOCK, "mock_cuda.cc"), os.path.join(HERE, "simt_emu.cc"), os.path.join(HERE, "emu_runtime.cc")]


def _digest(extra):
    h = hashlib.sha256(extra.encode())
    for root in (HOST, CSRC, os.path.join(ROOT, "include"), MOCK, HERE):
        for f in sorted(os.listdir(root)):
            p = os.path.join(root, f)
            if os.path.isfile(p) and f.endswith((".cc", ".cu", ".h", ".py")):
                h.update(p.encode())
                h.update(open(p, "rb").read())
    return h.hexdigest()[:16]


MUTATIONS = {
    # planted bugs for the checks that are supposed to find them (tools/sanitize_ingest.sh, tests/test_launch_shapes_mutants.py):
    # name -> (file under csrc/, old text, new text)
    "copies_do_not_wait_for_the_callers_stream": ("host/gpu_reader.cu", "for (auto cs : G.copy_streams) CU_TRY(cudaStreamWaitEvent(cs, G.entry_ev, 0));",
                                                   "/* planted: the copy streams start without waiting for what the caller enqueued before the read */;"),
    "callers_stream_does_not_wait_for_the_read": ("host/gpu_reader.cu", "CU_TRY(cudaStreamWaitEvent(caller, G.done_ev, 0));",
                                                   "/* planted: the caller's stream continues without waiting for the read */;"),
    "verifier_does_not_wait_for_the_copy": ("host/gpu_reader.cu", "cudaStreamWaitEvent(G.vstream, G.copy_ev[super_slot(g)], 0);", "/* planted: the verify stream no longer waits for the group's copies */;"),
    # K5's scale walk divides view positions in 32 bits even when a position or the view's width is >= 2^32
    "scale_walk_divides_in_32_bits": ("kernels.cu", "{ return (a | b) >> 32 ? a / b : uint64_t(uint32_t(a) / uint32_t(b)); }",
                                      "{ return uint64_t(uint32_t(a) / uint32_t(b)); /* planted: always 32-bit */ }"),
    # the shifted walk loses its row count above 1023 rows of 512 bytes: wrong only for segments of >= 512 KiB (s >= 19)
    "shifted_walk_drops_rows_past_1023": ("kernels.cu", "const uint32_t R = L >> 9, nv = (L & 511u) >> 4;\n    const uint32_t nvec = (L >> 4) + 1;",
                                          "const uint32_t R = (L >> 9) & 0x3ffu, nv = (L & 511u) >> 4;  /* planted */\n    const uint32_t nvec = (L >> 4) + 1;"),
    # K5's forward segment search gives up after 6 halvings: a grid stride that skips more than 64 segments lands short of its segment
    "cast_segment_search_spans_64_segments": ("kernels.cu", "            while (lo < hi) {\n                const uint32_t mid",
                                              "            for (int it = 0; lo < hi && it < 6; it++) {  /* planted */\n                const uint32_t mid"),
    # readv_device keeps a span's offset inside its range's destination in 32 bits: wrong for rows 4 GiB or more past the range's start
    "readv_row_offset_32_bits": ("host/gpu_reader.cu", "auto dst_of = [&](const ReadvSpan& s) { return rel(ranges[s.range].dst) + s.dst_off; };",
                                 "auto dst_of = [&](const ReadvSpan& s) { return rel(ranges[s.range].dst) + int64_t(uint32_t(s.dst_off)); /* planted */ };"),
    # the cast planner places the rest of an F16 -> F32 row that crosses a block edge at its source byte offset, not its destination one
    "cast_row_rest_offset_in_source_bytes": ("host/readv_plan.cc", "emit(q, take, 1, row * r.dst_pitch + col / ss * ds);",
                                             "emit(q, take, 1, row * r.dst_pitch + col / ss * (r.src_dtype == CV_DTYPE_F16 && r.dst_dtype == CV_DTYPE_F32 ? ss : ds));  /* planted */"),
    # the readv staging slots are spaced by the block length rounded down to 16 bytes: blocks whose length is not a multiple of 16
    # overlap their neighbour's slot
    "readv_stage_slots_rounded_down_to_16": ("host/gpu_reader.cu", "const int64_t at = rel(stage + slot * static_cast<size_t>(stage_block));",
                                             "const int64_t at = rel(stage + slot * static_cast<size_t>(stage_block & ~int64_t(15)));  /* planted */"),
    # K2's prefix checks (tests/test_kernel_verdicts_mutants.py): a frame of another RPC, of another request, or with a header in front
    # of its payload is accepted; a legal 16 MiB frame is rejected
    "k2_ignores_header_len": ("kernels.cu", "if (header_len != static_cast<int32_t>(d.header_len)) e |= CV_FERR_HEADER_LEN;", "/* planted: no header_len check */"),
    "k2_ignores_code": ("kernels.cu", "if (code != d.code) e |= CV_FERR_CODE;", "/* planted: no code check */"),
    "k2_ignores_total_len": ("kernels.cu", "if (int64_t(total_len) != int64_t(CV_HEAD_SIZE) + d.header_len + d.data_len) e |= CV_FERR_TOTAL_LEN;",
                             "/* planted: no total_len check */"),
    "k2_compares_req_id_low_words": ("kernels.cu", "if (req_id != d.req_id) e |= CV_FERR_REQ_ID;",
                                     "if (uint32_t(req_id) != uint32_t(d.req_id)) e |= CV_FERR_REQ_ID;  /* planted */"),
    "k2_rejects_16_mib_of_data": ("kernels.cu", "data_len > CV_MAX_DATA_SIZE) e |= CV_FERR_DATA_RANGE;", "data_len >= CV_MAX_DATA_SIZE) e |= CV_FERR_DATA_RANGE;  /* planted */"),
    # cvk_verify_crcs / _masked: one count per warp with a mismatch, skipped entries compared, a mask entry never cleared
    "verify_counts_warps": ("kernels.cu", "atomicAdd(n_bad, __popc(m));", "atomicAdd(n_bad, 1u);  /* planted */"),
    "verify_ignores_the_skip_mask": ("kernels.cu", "const bool bad = i < n && !(skip && skip[i]) && crc[i] != expect[i];",
                                     "const bool bad = i < n && crc[i] != expect[i];  /* planted */"),
    "verify_marks_only_mismatches": ("kernels.cu", "if (i < n && bad_mask) bad_mask[i] = bad;", "if (i < n && bad_mask && bad) bad_mask[i] = 1;  /* planted */"),
}


def _mutated(fname, text, mutate):
    """text of csrc/<fname>, with the planted bug `mutate` in it if that bug lives in this file"""
    if not mutate or MUTATIONS[mutate][0] != fname:
        return text
    _, old, new = MUTATIONS[mutate]
    if text.count(old) != 1:
        raise RuntimeError("mutation %s: the text to replace occurs %d times in %s" % (mutate, text.count(old), fname))
    return text.replace(old, new)


def build(sanitize: str = "", mutate: str = "") -> str:
    common = ["-g", "-std=c++17", "-fPIC", "-pthread", "-msse4.2", "-Wall", "-Wno-unknown-pragmas", "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-I", HOST]
    out_dir = os.path.join("/tmp", "cv_simt_emu_" + _digest(" ".join(common) + sanitize + mutate))
    lib = os.path.join(out_dir, "libcurvine_b200_emu.so")
    if os.path.exists(lib):
        return lib
    os.makedirs(out_dir, exist_ok=True)
    kern = os.path.join(out_dir, "kernels_rewritten.cc")
    text = rewrite(_mutated("kernels.cu", open(os.path.join(CSRC, "kernels.cu")).read(), mutate))
    # the rewritten copy sits in /tmp: its two relative includes are made absolute
    text = text.replace('#include "../../include/curvine_b200_kernels.h"', '#include "%s"' % os.path.join(ROOT, "include", "curvine_b200_kernels.h"))
    text = text.replace('#include "crc_gf.h"', '#include "%s"' % os.path.join(CSRC, "crc_gf.h"))
    with open(kern, "w") as f:
        f.write(text)
    san = ["-fsanitize=" + sanitize, "-fno-omit-frame-pointer"] if sanitize else []
    jobs = []
    srcs = sources()
    if mutate and MUTATIONS[mutate][0].startswith("host/"):
        fname = MUTATIONS[mutate][0]
        name = os.path.basename(fname)
        mutated = os.path.join(out_dir, "mutated_" + name)
        with open(mutated, "w") as f:  # its relative includes resolve through -I HOST below
            f.write(_mutated(fname, open(os.path.join(CSRC, fname)).read(), mutate))
        srcs = [mutated if os.path.basename(x) == name else x for x in srcs]
    for src in srcs:
        extra = ["-O1", "-I", MOCK] + san
        if sanitize == "thread" and os.path.basename(src) == "simt_emu.cc":
            extra = ["-O1", "-I", MOCK, "-DCV_EMU_TSAN"]  # the scheduler is not instrumented: it IS the ordering, stated through annotations
        jobs.append((src, extra))
    jobs.append((kern, ["-O2", "-I", HERE, "-Wno-unused-function", "-Wno-unused-variable", "-Wno-unused-but-set-variable"] + san))  # <cuda_runtime.h> = this directory's
    procs, objs = [], []
    for src, extra in jobs:
        obj = os.path.join(out_dir, os.path.basename(src) + ".o")
        objs.append(obj)
        procs.append((src, subprocess.Popen(["g++"] + common + extra + ["-x", "c++", "-c", src, "-o", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode:
            raise RuntimeError("g++ failed for %s:\n%s" % (src, out.decode()))
    link = ["g++", "-shared", "-Wl,-Bsymbolic", "-o", lib + ".tmp"] + objs + ["-lpthread", "-ldl", "-lrt"] + (["-fsanitize=" + sanitize] if sanitize else [])
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode:
        raise RuntimeError("link failed:\n" + r.stdout.decode())
    os.replace(lib + ".tmp", lib)
    return lib


def build_selftest(sanitize: str = "") -> str:
    """the shim's own known-answer program (selftest.cu) -> path of the executable"""
    out_dir = os.path.join("/tmp", "cv_simt_emu_selftest_" + _digest("selftest" + sanitize))
    exe = os.path.join(out_dir, "selftest")
    if os.path.exists(exe):
        return exe
    os.makedirs(out_dir, exist_ok=True)
    src = os.path.join(out_dir, "selftest_rewritten.cc")
    with open(src, "w") as f:
        f.write(rewrite(open(os.path.join(HERE, "selftest.cu")).read()))
    base = ["g++", "-O1", "-g", "-std=c++17", "-pthread", "-Wall", "-Wno-unknown-pragmas", "-I", HERE, "-I", os.path.join(ROOT, "include"), "-I", CSRC]
    san = ["-fsanitize=" + sanitize, "-fno-omit-frame-pointer"] if sanitize else []
    sched = os.path.join(out_dir, "simt_emu.o")
    cmds = [base + (["-DCV_EMU_TSAN"] if sanitize == "thread" else san) + ["-c", os.path.join(HERE, "simt_emu.cc"), "-o", sched],
            base + san + ["-x", "c++", src, os.path.join(MOCK, "mock_cuda.cc"), os.path.join(HERE, "emu_runtime.cc"), "-x", "none", sched, "-o", exe + ".tmp", "-lpthread"]]
    for cmd in cmds:
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
        if r.returncode:
            raise RuntimeError("selftest build failed:\n" + r.stdout.decode())
    os.replace(exe + ".tmp", exe)
    return exe


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--selftest":
        print(build_selftest(sys.argv[2] if len(sys.argv) > 2 else ""))
    elif len(sys.argv) > 1 and sys.argv[1] == "--show":
        sys.stdout.write(rewrite(open(os.path.join(CSRC, "kernels.cu")).read()))
    elif len(sys.argv) > 1 and sys.argv[1] == "--mutate":
        print(build(sys.argv[3] if len(sys.argv) > 3 else "", sys.argv[2]))  # --mutate <name> [sanitize]
    else:
        print(build(sys.argv[1] if len(sys.argv) > 1 else ""))
