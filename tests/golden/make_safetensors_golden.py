"""safetensors checkpoints whose bytes come from the format's official writer, without that writer at test time.

Each checkpoint of CHECKPOINTS is a list of tensors with seeded contents (tensor_bytes).  Run with the `safetensors` package installed,
this script builds every checkpoint as torch tensors, serializes it with safetensors.torch.save, and records in
safetensors_official.json only what the writer decided: the header bytes (length prefix, JSON, padding), the spec, and the SHA-256
of the whole file.  rebuild() puts a file back together from the recorded header and the seeded tensor bytes at the header's
data_offsets; its SHA-256 must equal the recorded one, so the rebuilt bytes are the official writer's.

    python tests/golden/make_safetensors_golden.py           # write safetensors_official.json
    python tests/golden/make_safetensors_golden.py --check   # regenerate and fail on any difference from the committed file
"""
import hashlib
import json
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
JSON = os.path.join(HERE, "safetensors_official.json")

# bytes per element of the dtypes the specs use (F4: two elements per byte)
SIZE = {"F8_E4M3": 1, "F8_E5M2": 1, "F8_E8M0": 1, "F32": 4, "F16": 2, "BF16": 2, "I64": 8, "I32": 4, "U16": 2, "U8": 1, "BOOL": 1, "C64": 8}


def _w(name, dt, shape, scale=None):
    """a tensor spec; `scale` = (dtype, shape) of the weight's scale tensor, named name + "_scale" """
    return [name, dt, list(shape)] + ([[name + "_scale", scale[0], list(scale[1])]] if scale else [])


def _grid(R, C, block):
    return (-(-R // block[0]), -(-C // block[1]))


def _checkpoints():
    """name -> {"scale_block", "tensors": [[name, dtype, shape], ...], "scales": {weight: scale}}.  R and C of the 2-D FP8 weights are
    drawn from {1, 7, 127, 128, 129, 300}; small tensors sit between large ones so that several tensors share a block."""
    out = {}

    def add(key, block, specs):
        tensors, scales = [], {}
        for s in specs:
            tensors.append(s[:3])
            if len(s) == 4:
                tensors.append(s[3])
                scales[s[0]] = s[3][0]
        out[key] = {"scale_block": list(block), "tensors": tensors, "scales": scales}

    b = (128, 128)
    add("tiles_128x128", b, [
        _w("q.weight", "F8_E4M3", (129, 300), ("F32", _grid(129, 300, b))),
        ["one.i32", "I32", [1]],
        _w("k.weight", "F8_E5M2", (300, 129), ("BF16", _grid(300, 129, b))),
        ["empty.u16", "U16", [0, 5]],
        _w("v.weight", "F8_E4M3", (127, 7), ("F16", (127, 1))),
        ["scalar.u8", "U8", []],
        _w("o.weight", "F8_E5M2", (7, 1), ("F32", ())),
        _w("experts.w", "F8_E4M3", (3, 7, 129), ("BF16", (1,))),
        ["norm.f32", "F32", [33, 129]], ["norm.f16", "F16", [7, 300]], ["norm.bf16", "BF16", [129, 7]],
        ["ids.i64", "I64", [7, 3]], ["mask", "BOOL", [3, 1]],
        ["mx.scales", "F8_E8M0", [4, 7]], ["mx.f4", "F4", [5, 6]], ["rope.c64", "C64", [3]],
    ])
    b = (1, 16)
    add("rows_1x16", b, [
        _w("up.weight", "F8_E4M3", (1, 300), ("F16", _grid(1, 300, b))),
        ["scalar.i64", "I64", []],
        _w("down.weight", "F8_E5M2", (7, 127), ("F32", _grid(7, 127, b))),
        _w("gate.weight", "F8_E4M3", (128, 129), ("BF16", (128, 1))),
        ["empty.f32", "F32", [3, 0]],
        _w("lm.weight", "F8_E5M2", (129, 1), ("F16", (1,))),
        ["embed.bf16", "BF16", [300, 7]], ["ln.f16", "F16", [129]], ["bias.f32", "F32", [127, 7]],
        ["pos.i32", "I32", [7, 7]], ["tok.u16", "U16", [129]], ["one.u8", "U8", [1]], ["keep", "BOOL", [7, 128]],
    ])
    b = (3, 7)
    add("tiles_3x7", b, [
        _w("wq", "F8_E4M3", (300, 127), ("BF16", _grid(300, 127, b))),
        ["one.bool", "BOOL", [1]],
        _w("wk", "F8_E5M2", (129, 7), ("F32", _grid(129, 7, b))),
        _w("wv", "F8_E4M3", (1, 1), ("BF16", ())),
        _w("moe", "F8_E5M2", (2, 3, 127), ("F16", (1,))),
        ["h.f16", "F16", [128, 7]], ["h.bf16", "BF16", [7, 129]], ["h.f32", "F32", [1, 300]],
        ["n.i64", "I64", [1]], ["e.u8", "U8", [0]], ["mx.e8m0", "F8_E8M0", [129]], ["freqs.c64", "C64", [7, 2]],
    ])
    b = (64, 48)
    add("tiles_64x48", b, [
        _w("big", "F8_E5M2", (300, 300), ("F16", _grid(300, 300, b))),
        ["z.i32", "I32", []],
        _w("mid", "F8_E4M3", (129, 128), ("F32", _grid(129, 128, b))),
        ["zz.bool", "BOOL", [0]],
        _w("small", "F8_E4M3", (7, 127), ("F32", (7, 1))),
        ["s.f32", "F32", [129, 1]], ["s.bf16", "BF16", [127]], ["s.f16", "F16", [300, 1]],
        ["c.u16", "U16", [7, 1]], ["c.i64", "I64", [0, 3]], ["fp4", "F4", [7, 128]],
    ])
    return out


CHECKPOINTS = _checkpoints()

# float32 bit patterns at the edges of the conversions: bfloat16 and float16 rounding ties (the dropped bits exactly half, and one
# either side), values that overflow float16 and bfloat16, float16 subnormals and the float32 subnormals, zeros, infinities, NaNs
_F32_EDGES = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00001, 0x7F800001, 0x7F7FFFFF, 0xFF7FFFFF, 0x00000001,
              0x807FFFFF, 0x00800000, 0x3F808000, 0x3F818000, 0x3F807FFF, 0x3F808001, 0x7F7F8000, 0x7F7F7FFF, 0x477FE000, 0x477FF000,
              0x477FEFFF, 0x477FF001, 0x47800000, 0xC7800000, 0x38800000, 0x387FF000, 0x33000000, 0x33000001, 0x33800000, 0x3F801000,
              0x3F803000, 0x3F800FFF, 0x3F801001, 0x36A00000, 0x36A01000, 0x80000001]
# float16 and bfloat16 patterns: subnormals, the largest finite values, infinities, NaNs, values whose conversion rounds a tie
_F16_EDGES = [0x0000, 0x8000, 0x0001, 0x03FF, 0x0400, 0x7BFF, 0x7C00, 0xFC00, 0x7C01, 0x7E00, 0xFFFF, 0x3C00, 0x3C01, 0x8001]
_BF16_EDGES = [0x0000, 0x8000, 0x0001, 0x007F, 0x0080, 0x7F7F, 0xFF7F, 0x7F80, 0xFF80, 0x7F81, 0x7FC0, 0x477F, 0x4780, 0x3380, 0x3381,
               0x387F, 0x3880, 0x3F81, 0xC77F, 0x33C0]


def _seed(ck, name):
    return int.from_bytes(hashlib.sha256(("%s/%s" % (ck, name)).encode()).digest()[:8], "little")


def _numel(shape):
    n = 1
    for d in shape:
        n *= d
    return n


def nbytes(dt, shape):
    n = _numel(shape)
    return (n + 1) // 2 if dt == "F4" else n * SIZE[dt]


def tensor_bytes(ck, name, dt, shape, is_scale=False):
    """the seeded contents of tensor `name` of checkpoint `ck` -> bytes"""
    rng = np.random.default_rng(_seed(ck, name))
    n = _numel(shape)
    if dt in ("F8_E4M3", "F8_E5M2"):  # every one of the 256 patterns once (NaNs included) when there is room, then random bytes
        raw = np.resize(rng.permutation(256).astype(np.uint8), n) if n >= 256 else rng.integers(0, 256, n).astype(np.uint8)
        if n > 256:
            raw[256:] = rng.integers(0, 256, n - 256)
        return raw.tobytes()
    if is_scale:  # magnitudes 2^-24 .. 2^8 of both signs, so that products round, underflow and (into float16) overflow
        v = np.ldexp(rng.uniform(0.5, 1.0, n), rng.integers(-24, 9, n)) * np.where(rng.random(n) < 0.25, -1.0, 1.0)
        f32 = v.astype(np.float32)
        if dt == "F32":
            return f32.tobytes()
        if dt == "F16":
            return f32.astype(np.float16).tobytes()
        return (f32.view(np.uint32) >> 16).astype(np.uint16).tobytes()  # BF16: the high half
    if dt in ("F32", "F16", "BF16"):  # random bit patterns, most of them ordinary values, with the edges salted in
        if dt == "F32":
            v = (rng.standard_normal(n) * np.ldexp(1.0, rng.integers(-20, 20, n))).astype(np.float32).view(np.uint32)
            edges, width = _F32_EDGES, np.uint32
        else:
            v = rng.standard_normal(n).astype(np.float32) * np.float32(300)
            v = v.astype(np.float16).view(np.uint16) if dt == "F16" else (v.view(np.uint32) >> 16).astype(np.uint16)
            edges, width = (_F16_EDGES if dt == "F16" else _BF16_EDGES), np.uint16
        v = v.astype(width)
        rand = rng.random(n) < 0.2
        v[rand] = rng.integers(0, np.iinfo(width).max, int(rand.sum()), endpoint=True).astype(width)
        k = rng.permutation(n)[:len(edges)]
        v[k] = np.array(edges, dtype=np.uint64)[:k.size].astype(width)
        return v.tobytes()
    if dt == "BOOL":
        return rng.integers(0, 2, n).astype(np.uint8).tobytes()
    if dt == "C64":
        return rng.standard_normal(2 * n).astype(np.float32).tobytes()
    return rng.integers(0, 256, nbytes(dt, shape)).astype(np.uint8).tobytes()  # integers, F8_E8M0, F4


def contents(ck):
    """{tensor name: (dtype, shape, bytes)} of checkpoint `ck`"""
    spec = CHECKPOINTS[ck]
    scale_names = set(spec["scales"].values())
    return {name: (dt, tuple(shape), tensor_bytes(ck, name, dt, shape, name in scale_names)) for name, dt, shape in spec["tensors"]}


def official_file(ck):
    """checkpoint `ck` serialized by safetensors.torch.save -> bytes (needs the safetensors package)"""
    import torch
    from safetensors.torch import save
    tdt = {"F8_E4M3": torch.float8_e4m3fn, "F8_E5M2": torch.float8_e5m2, "F8_E8M0": torch.float8_e8m0fnu, "F32": torch.float32,
           "F16": torch.float16, "BF16": torch.bfloat16, "I64": torch.int64, "I32": torch.int32, "U16": torch.uint16, "U8": torch.uint8,
           "BOOL": torch.bool, "C64": torch.complex64}
    tensors = {}
    for name, (dt, shape, raw) in contents(ck).items():
        u8 = torch.frombuffer(bytearray(raw), dtype=torch.uint8) if raw else torch.empty(0, dtype=torch.uint8)
        if dt == "F4":  # torch holds F4 as pairs of elements per byte: the last dimension halves
            assert shape[-1] % 2 == 0
            tensors[name] = u8.view(torch.float4_e2m1fn_x2).reshape(shape[:-1] + (shape[-1] // 2,))
        else:
            tensors[name] = u8.view(tdt[dt]).reshape(shape)
    return save(tensors)


def header_of(blob):
    (n,) = struct.unpack("<Q", blob[:8])
    return blob[:8 + n]


def rebuild(ck, header_hex):
    """the official file of checkpoint `ck` from its recorded header bytes and the seeded tensor bytes -> bytes"""
    head = bytes.fromhex(header_hex)
    header = json.loads(head[8:].decode())
    data = bytearray(max([e["data_offsets"][1] for k, e in header.items() if k != "__metadata__"] + [0]))
    for name, (dt, shape, raw) in contents(ck).items():
        b, e = header[name]["data_offsets"]
        assert e - b == len(raw) and header[name]["dtype"] == dt and tuple(header[name]["shape"]) == shape, name
        data[b:e] = raw
    return head + bytes(data)


def load():
    """the committed record: {checkpoint: {"spec", "header", "sha256", "size"}}"""
    with open(JSON) as f:
        return json.load(f)


def generate():
    out = {"checkpoints": {}}
    for ck in CHECKPOINTS:
        blob = official_file(ck)
        out["checkpoints"][ck] = {"spec": CHECKPOINTS[ck], "header": header_of(blob).hex(), "sha256": hashlib.sha256(blob).hexdigest(),
                                  "size": len(blob)}
        assert rebuild(ck, out["checkpoints"][ck]["header"]) == blob, ck
    return json.dumps(out, indent=1, sort_keys=True) + "\n"


if __name__ == "__main__":
    text = generate()
    if "--check" in sys.argv[1:]:
        with open(JSON) as f:
            old = f.read()
        if old != text:
            sys.exit("safetensors_official.json differs from what the installed safetensors writes")
        print("safetensors_official.json: every header and hash reproduced")
    else:
        with open(JSON, "w") as f:
            f.write(text)
        print("wrote", JSON)
