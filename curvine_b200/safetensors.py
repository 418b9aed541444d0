"""safetensors checkpoints straight into HBM: every tensor of the file (or a named subset) in its own CUDA tensor, from ONE vectored
device read (Reader.readv_device) in which every block the tensors touch is CRC-verified whole on the GPU.

The format needs no dependency: an 8-byte little-endian header length, a JSON object mapping each tensor name to
{"dtype", "shape", "data_offsets": [begin, end]} (offsets relative to the first byte after the header), an optional "__metadata__"
entry, then the raw little-endian tensor bytes."""
import json
import numbers
import struct
from typing import Callable, Dict, Iterable, List, Optional, Tuple

from . import _lib
from . import fs as _fs

# the safetensors reference reader refuses headers larger than this; a larger length is a corrupt or hostile file
MAX_HEADER_BYTES = 100 << 20


class SafetensorsError(ValueError):
    """The file is not a well-formed safetensors file."""


# every dtype of the format -> its width in bits.  F4 and F6_* pack their elements into bytes, so a tensor of theirs must end on a
# byte boundary (numel * bits a multiple of 8), as the format's own reader requires
BITS = {"F4": 4, "F6_E2M3": 6, "F6_E3M2": 6, "BOOL": 8, "U8": 8, "I8": 8, "F8_E4M3": 8, "F8_E5M2": 8, "F8_E8M0": 8, "I16": 16, "U16": 16,
        "F16": 16, "BF16": 16, "I32": 32, "U32": 32, "F32": 32, "I64": 64, "U64": 64, "F64": 64, "C64": 64}


def dtypes() -> dict:
    """safetensors dtype name -> torch dtype, for every dtype of the format this torch build has."""
    import torch
    m = {"F64": torch.float64, "F32": torch.float32, "F16": torch.float16, "BF16": torch.bfloat16, "I64": torch.int64, "I32": torch.int32,
         "I16": torch.int16, "I8": torch.int8, "U8": torch.uint8, "BOOL": torch.bool, "F8_E4M3": torch.float8_e4m3fn,
         "F8_E5M2": torch.float8_e5m2}
    for name, attr in (("U16", "uint16"), ("U32", "uint32"), ("U64", "uint64"), ("F8_E8M0", "float8_e8m0fnu"), ("C64", "complex64")):
        if hasattr(torch, attr):
            m[name] = getattr(torch, attr)
    return m


def _is_int(x) -> bool:
    return isinstance(x, int) and not isinstance(x, bool)


def parse_header(read: Callable[[int, int], bytes], file_len: int) -> Tuple[int, Dict[str, tuple]]:
    """Reads and validates the header of a safetensors file of `file_len` bytes; `read(off, n)` returns n bytes of the file at off.
    -> (data_start, {name: (torch dtype, shape, begin, end)}) with begin/end relative to data_start; a tensor of a dtype of the format
    that torch cannot hold (F4, F6_E2M3, F6_E3M2) has the format's name in place of the torch dtype.  Every dtype of the format
    parses; a tensor's shape must need exactly its bytes, numel * bits = 8 * (end - begin).  Unlike the format's own reader, this one
    allows gaps between tensors and after the last one.  Raises SafetensorsError."""
    if file_len < 8:
        raise SafetensorsError("file of %d bytes is too short for the 8-byte header length" % file_len)
    (n,) = struct.unpack("<Q", read(0, 8))
    if n > MAX_HEADER_BYTES:
        raise SafetensorsError("header length %d exceeds the %d-byte limit" % (n, MAX_HEADER_BYTES))
    if 8 + n > file_len:
        raise SafetensorsError("header length %d runs past the end of a %d-byte file" % (n, file_len))
    try:
        header = json.loads(read(8, n).decode("utf-8"))
    except (UnicodeDecodeError, ValueError, RecursionError) as e:
        raise SafetensorsError("header is not valid JSON: %s" % e)
    if not isinstance(header, dict):
        raise SafetensorsError("header is not a JSON object")
    data_start, data_len = 8 + n, file_len - 8 - n
    table = dtypes()
    out = {}
    for name, ent in header.items():
        if name == "__metadata__":
            continue
        if not isinstance(ent, dict):
            raise SafetensorsError("%s: entry is not an object" % name)
        dt, shape, offs = ent.get("dtype"), ent.get("shape"), ent.get("data_offsets")
        if not isinstance(dt, str) or dt not in BITS:
            raise SafetensorsError("%s: unknown dtype %r" % (name, dt))
        if not isinstance(shape, list) or not all(_is_int(d) and d >= 0 for d in shape):
            raise SafetensorsError("%s: shape %r is not a list of non-negative integers" % (name, shape))
        if not isinstance(offs, list) or len(offs) != 2 or not all(_is_int(o) for o in offs):
            raise SafetensorsError("%s: data_offsets %r is not a pair of integers" % (name, offs))
        begin, end = offs
        if not 0 <= begin <= end <= data_len:
            raise SafetensorsError("%s: data_offsets [%d, %d) lie outside the %d-byte data section" % (name, begin, end, data_len))
        count = 1
        for d in shape:
            count *= d
        need = count * BITS[dt]
        if need % 8:
            raise SafetensorsError("%s: shape %r of %s is %d bits, which does not end on a byte boundary" % (name, shape, dt, need))
        if need != 8 * (end - begin):
            raise SafetensorsError("%s: shape %r of %s needs %d bytes, data_offsets hold %d" % (name, shape, dt, need // 8, end - begin))
        out[name] = (table.get(dt, dt), tuple(shape), begin, end)
    spans = sorted((b, e, name) for name, (_, _, b, e) in out.items() if e > b)
    for (_, e0, n0), (b1, _, n1) in zip(spans, spans[1:]):
        if b1 < e0:
            raise SafetensorsError("tensors %s and %s overlap in the data section" % (n0, n1))
    return data_start, out


def _open_header(fs, path):
    """-> (reader, data_start, entries) of safetensors file `path`; the caller completes the reader."""
    r = fs.open(path)

    def read(off, n):
        r.seek(off)
        b = r.read_full(n)
        if len(b) != n:
            raise SafetensorsError("short read of the header: %d of %d bytes" % (len(b), n))
        return b

    try:
        data_start, entries = parse_header(read, r.len())
    except BaseException:
        r.complete()
        raise
    return r, data_start, entries


def read_header(fs: "_fs.CurvineFileSystem", path: str) -> Dict[str, tuple]:
    """{name: (torch dtype, shape)} of safetensors file `path`, from its header alone: what a tensor-parallel rank needs to compute the
    `slices` it passes to load_file.  A tensor whose dtype torch cannot hold (F4, F6_E2M3, F6_E3M2) is listed with the format's dtype
    name in place of the torch dtype; load_file refuses to load it."""
    r, _, entries = _open_header(fs, path)
    r.complete()
    return {name: (dt, shape) for name, (dt, shape, _, _) in entries.items()}


def _is_integral(x) -> bool:
    return isinstance(x, numbers.Integral) and not isinstance(x, bool)


def _dtypes_of(codes) -> tuple:
    """the torch dtypes whose cast-read code (fs.cast_dtype_codes) is one of `codes`"""
    return tuple(t for t, c in _fs.cast_dtype_codes().items() if c in codes)


def _cast_targets(data_start: int, entries: Dict[str, tuple], selected, dtype, scaled=()) -> Dict[str, object]:
    """{name: dtype of the result} for load_file(dtype=...): the float32, float16 and bfloat16 tensors become `dtype`, the others stay as
    stored.  Raises ValueError for a target dtype other than those three, for a selected float tensor of another width (float64, float8:
    not converted) and for a converting tensor whose data offset is not a multiple of its element size.  The float8 weights named in
    `scaled` (load_file(scales=...)) become `dtype` too."""
    floats = _dtypes_of(_lib.FLOAT_CODES)
    if dtype not in floats:
        raise ValueError("dtype %s: loads convert to float32, float16 or bfloat16 only" % (dtype,))
    out = {}
    for name in selected:
        stored, _, begin, end = entries[name]
        if name in scaled:
            out[name] = dtype
            continue
        if stored.is_floating_point and stored not in floats:
            raise ValueError("%s: %s tensors are not converted on load (only float32, float16 and bfloat16 are)" % (name, stored))
        out[name] = dtype if stored in floats else stored
        if out[name] != stored and (data_start + begin) % stored.itemsize:
            raise ValueError("%s: data offset %d is not a multiple of its %d-byte element size" % (name, data_start + begin, stored.itemsize))
    return out


def _scale_geometry(entries: Dict[str, tuple], selected, scales, scale_block, dtype) -> Dict[str, tuple]:
    """{weight: (scale name, scale_rows, scale_cols, block_rows, block_cols, cols)} for the selected weights of load_file(scales=...).
    The weight is seen as the row-major 2-D view [V_rows, cols = shape[-1]]; its scale is one element (per tensor, any shape), (V_rows, 1)
    for a 2-D weight (per row), or, with scale_block = (br, bc), (ceil(R / br), ceil(C / bc)) for a 2-D weight (blocks).  Raises
    ValueError, naming the weight and its scale, for anything else (see load_file)."""
    if dtype is None:
        raise ValueError("scales are given without dtype: dequantized weights need a result dtype")
    if scale_block is not None and (not isinstance(scale_block, (tuple, list)) or len(scale_block) != 2
                                    or not all(_is_integral(x) and x >= 1 for x in scale_block)):
        raise ValueError("scale_block %r is not (block_rows, block_cols) of positive integers" % (scale_block,))
    f8, floats = _dtypes_of(_lib.F8_CODES), _dtypes_of(_lib.FLOAT_CODES)
    sel = set(selected)
    out = {}
    for w, sname in dict(scales).items():
        if w not in entries:
            raise ValueError("%s (scale %s): the file holds no such weight" % (w, sname))
        if sname not in entries:
            raise ValueError("%s: its scale %s is not in the file" % (w, sname))
        if sname == w or sname in scales:
            raise ValueError("%s: its scale %s is itself a weight named in scales" % (w, sname))
        wdt, wshape, _, _ = entries[w]
        sdt, sshape, _, _ = entries[sname]
        if wdt not in f8:
            raise ValueError("%s (scale %s): a scaled weight must be F8_E4M3 or F8_E5M2, not %s" % (w, sname, wdt))
        if sdt not in floats:
            raise ValueError("%s: its scale %s must be F32, F16 or BF16, not %s" % (w, sname, sdt))
        if w not in sel:
            continue
        cols = wshape[-1] if wshape else 1
        numel = 1
        for x in wshape:
            numel *= x
        vrows = numel // cols if cols else 0
        snumel = 1
        for x in sshape:
            snumel *= x
        if snumel == 1:  # per tensor
            out[w] = (sname, 1, 1, max(1, vrows), max(1, cols), max(1, cols))
        elif len(wshape) == 2 and tuple(sshape) == (wshape[0], 1):  # per row
            out[w] = (sname, wshape[0], 1, 1, max(1, cols), max(1, cols))
        elif len(wshape) == 2 and scale_block is not None and tuple(sshape) == (-(-wshape[0] // scale_block[0]), -(-wshape[1] // scale_block[1])):
            out[w] = (sname, sshape[0], sshape[1], int(scale_block[0]), int(scale_block[1]), max(1, cols))
        else:
            raise ValueError("%s %s: its scale %s has shape %s, which is neither one element, (rows, 1) of a 2-D weight nor the "
                             "(ceil(R / br), ceil(C / bc)) blocks of scale_block=%s" % (w, tuple(wshape), sname, tuple(sshape), scale_block))
    return out


def plan_ranges(data_start: int, entries: Dict[str, tuple], selected, slices=None, dtype=None, scales=None, scale_block=None) -> List[tuple]:
    """The loader's ranges, without a GPU.  -> [(name, dtype, shape of the result, range)] for the selected names, in order, where range
    is (file_off, row_len, rows, file_pitch, dst_pitch) of Reader.readv_strided_device (d_ptr left out), or None when the tensor has no
    bytes to read.  An unsliced tensor is one row.  slices[name] = (dim, start, stop) keeps [start, stop) of dimension dim: the rows are
    the prod(shape[:dim]) pieces of the row-major tensor that hold it, each (stop - start) * inner bytes long and shape[dim] * inner bytes
    apart (inner = prod(shape[dim+1:]) * itemsize), landing back to back.  With `dtype` (float32, float16 or bfloat16) the float32,
    float16 and bfloat16 tensors come back in `dtype`, the others as stored: dtype is the result's and range is (file_off, row_len, rows,
    file_pitch, dst_pitch, stored dtype, result dtype) of Reader.readv_cast_device, its file side in stored bytes and its dst_pitch in
    result bytes.  With `scales` ({float8 weight: name of its scale tensor}, dtype required; scale_block = (br, bc) for block scales)
    every range gets one more item, the `scale` of Reader.readv_scaled_device with the scale tensor's NAME in place of its pointer: None,
    or (scale name, scale_rows, scale_cols, block_rows, block_cols, cols, first_elem), first_elem being a sliced weight's offset in the
    full tensor in elements.  Raises KeyError for a sliced name the file does not hold, ValueError for a selected tensor whose dtype
    torch cannot hold (see parse_header), a malformed slice, a sliced name outside `selected`, a tensor load_file(dtype=...) cannot
    convert (see _cast_targets) or a weight and scale load_file(scales=...) cannot dequantize (see _scale_geometry)."""
    for name in selected:
        if isinstance(entries[name][0], str):
            raise ValueError("%s: its dtype %s has no torch dtype, so it cannot be loaded" % (name, entries[name][0]))
    slices = dict(slices or {})
    sel = set(selected)
    if scale_block is not None and scales is None:
        raise ValueError("scale_block is given without scales")
    geo = _scale_geometry(entries, selected, scales, scale_block, dtype) if scales is not None else None
    targets = _cast_targets(data_start, entries, selected, dtype, geo or ()) if dtype is not None else None
    for name, spec in slices.items():
        if name not in entries:
            raise KeyError("the file holds no tensor named %r" % (name,))
        if name not in sel:
            raise ValueError("%s is sliced but not among the selected names" % name)
        if not isinstance(spec, (tuple, list)) or len(spec) != 3 or not all(_is_integral(x) for x in spec):
            raise ValueError("%s: slice %r is not (dim, start, stop) of integers" % (name, spec))
        shape = entries[name][1]
        dim, start, stop = (int(x) for x in spec)
        if not shape:
            raise ValueError("%s: a 0-d tensor cannot be sliced" % name)
        if not -len(shape) <= dim < len(shape):
            raise ValueError("%s: dim %d is out of range for a %d-d tensor" % (name, dim, len(shape)))
        d = dim % len(shape)
        if not 0 <= start <= stop <= shape[d]:
            raise ValueError("%s: [%d, %d) is not a slice of dimension %d of size %d" % (name, start, stop, dim, shape[d]))
    out = []
    for name in selected:
        stored, shape, begin, end = entries[name]
        dt = targets[name] if targets is not None else stored
        tail = (stored, dt) if targets is not None else ()  # the dtypes of a readv_cast_device range
        if geo is not None:  # and the scale of a readv_scaled_device range
            tail += (geo[name] + (0,) if name in geo else None,)
        if name not in slices:
            out.append((name, dt, shape, (data_start + begin, end - begin, 1, 0, 0) + tail if end > begin else None))
            continue
        dim, start, stop = (int(x) for x in slices[name])
        d = dim % len(shape)
        inner = 1  # elements
        for x in shape[d + 1:]:
            inner *= x
        rows = 1
        for x in shape[:d]:
            rows *= x
        row_len = (stop - start) * inner * stored.itemsize
        res = shape[:d] + (stop - start,) + shape[d + 1:]
        if geo is not None and name in geo:  # the slice's first element in the full tensor
            tail = tail[:-1] + (geo[name] + (start * inner,),)
        rng = (data_start + begin + start * inner * stored.itemsize, row_len, rows, shape[d] * inner * stored.itemsize,
               (stop - start) * inner * dt.itemsize) + tail if row_len and rows else None
        out.append((name, dt, res, rng))
    return out


def load_file(fs: "_fs.CurvineFileSystem", path: str, device=None, names: Optional[Iterable[str]] = None,
              verify: bool = True, slices: Optional[Dict[str, tuple]] = None, dtype=None, scales: Optional[Dict[str, str]] = None,
              scale_block: Optional[tuple] = None) -> Dict[str, "object"]:
    """The tensors of safetensors file `path` (all of them, or those in `names`) as tensors on `device` (default: the current CUDA
    device).  One vectored read moves them: blocks that no selected tensor touches are not fetched, and every touched block is
    CRC-verified whole, including the bytes of unselected neighbours that share it.  `slices` maps a name to (dim, start, stop): that
    tensor comes back contiguous with shape[dim] = stop - start -- a tensor-parallel rank's shard, without the rest of the tensor ever
    reaching HBM (see plan_ranges).  `dtype` (torch.float32, torch.float16 or torch.bfloat16) converts every float32, float16 and bfloat16
    tensor to it on the GPU in the same read, bit-identical to Tensor.to() on the CPU; integer, bool and complex64 tensors come back as
    stored, and a selected float tensor of another width (float64, float8 including F8_E8M0) is refused.  The
    stored copy never exists in HBM: a converted tensor's blocks pass through the reader's bounded staging.  `scales` maps float8 weights
    (F8_E4M3, F8_E5M2) to the names of their scale tensors in the same file (F32, F16 or BF16: one element, one per row of a 2-D weight,
    or with scale_block = (br, bc) one per br x bc tile): those weights come back in `dtype`, dequantized on the GPU as they load, each
    element (x.float() * scale.float()).to(dtype) bit for bit; they compose with `slices`.  The scales are read first, as stored, into
    temporaries; the second read then dequantizes (two calls on the caller's stream, one verification).  Float8 tensors not named in
    `scales` are refused, as without it.  Without `dtype` every tensor comes back as stored, F8_E8M0 as float8_e8m0fnu and C64 as
    complex64.  Raises IOError when a block fails verification and `verify` is set, SafetensorsError for a malformed header, KeyError for
    a name the file does not hold, ValueError for a selected tensor whose dtype torch cannot hold (F4, F6_E2M3, F6_E3M2; names=None
    selects them too), a malformed slice, a tensor `dtype` cannot convert or a weight and scale that cannot be dequantized (all before
    anything is allocated or read)."""
    import torch
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    r, data_start, entries = _open_header(fs, path)
    try:
        selected = list(entries) if names is None else list(dict.fromkeys(names))
        for name in selected:
            if name not in entries:
                raise KeyError("%s holds no tensor named %r" % (path, name))
        plan = plan_ranges(data_start, entries, selected, slices, dtype, scales, scale_block)
        stream = torch.cuda.current_stream(dev).cuda_stream
        d_scales = {}  # scale name -> the scale tensor as stored, read by the first of the two calls
        if scales is not None:
            for sname in dict.fromkeys(rng[7][0] for _, _, _, rng in plan if rng is not None and rng[7] is not None):
                sdt, sshape, begin, end = entries[sname]
                d_scales[sname] = torch.empty((end - begin) // sdt.itemsize, dtype=sdt, device=dev)
            r.readv_strided_device([(data_start + entries[n][2], entries[n][3] - entries[n][2], 1, 0, t.data_ptr(), 0)
                                    for n, t in d_scales.items() if t.numel()], stream)
        out, ranges = {}, []
        for name, dt, shape, rng in plan:
            t = torch.empty(shape, dtype=dt, device=dev)
            out[name] = t
            if rng is not None:
                file_off, row_len, rows, file_pitch, dst_pitch = rng[:5]
                tail = tuple(rng[5:])
                if scales is not None and tail[2] is not None:  # the scale tensor's name -> its temporary
                    sc = d_scales[tail[2][0]]
                    tail = tail[:2] + ((sc.data_ptr(), sc.dtype) + tuple(tail[2][1:]),)
                ranges.append((file_off, row_len, rows, file_pitch, t.data_ptr(), dst_pitch) + tail)
        if dtype is None:
            r.readv_strided_device(ranges, stream)
        elif scales is None:  # one call still: the ranges that convert nothing have src == dst, and their whole blocks land in place
            r.readv_cast_device(ranges, stream)
        else:  # ordered after the scales' read on `stream`: each call waits for the stream at entry and makes it wait at exit
            r.readv_scaled_device(ranges, stream)
        _, bad, _ = r.verify()
        if verify and bad:
            raise IOError("%d blocks of %s failed CRC verification" % (bad, path))
        return out
    finally:
        r.complete()
