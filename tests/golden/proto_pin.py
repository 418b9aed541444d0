"""An INDEPENDENT proto2 encoder for the block-path headers: google.protobuf with descriptors built at run time (no protoc
in the image).  Test infrastructure: pins the byte-level restatements in oracle/wire.py and curvine_b200/csrc/host/wire.cc
against a third implementation of the protobuf wire format, so that the header bytes are no longer checked only against
themselves (VERDICT r1: "frame/protobuf bytes: parity unpinned").

The message shapes are restated from the reference's .proto files, field by field (paths relative to the CurvineIO/curvine source tree):
    curvine-common/proto/worker.proto:10-18   BlockWriteRequest
    curvine-common/proto/worker.proto:27-34   BlockWriteResponse       (pipeline_status, field 6, is not on this path: omitted)
    curvine-common/proto/worker.proto:38-47   BlockReadRequest
    curvine-common/proto/worker.proto:49-54   BlockReadResponse
    curvine-common/proto/worker.proto:56-60   DataHeaderProto
    curvine-common/proto/common.proto:98-104  ExtendedBlockProto       (alloc_opts, field 5, optional and never set here: omitted)
    curvine-common/proto/common.proto:9-16    StorageTypeProto
    curvine-common/proto/common.proto:31-38   FileTypeProto
prost 0.11 (Cargo.toml:67) writes a proto2 `required` field always, defaults included; google.protobuf does the same for a
required field that has been SET, so every required field is set explicitly by `build()`.
"""
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

F = descriptor_pb2.FieldDescriptorProto
REQ, OPT = F.LABEL_REQUIRED, F.LABEL_OPTIONAL


def _field(msg, name, number, ftype, label=REQ, type_name=None, default=None):
    f = msg.field.add()
    f.name, f.number, f.type, f.label = name, number, ftype, label
    if type_name:
        f.type_name = type_name
    if default is not None:
        f.default_value = default


def _file():
    fd = descriptor_pb2.FileDescriptorProto()
    fd.name, fd.package, fd.syntax = "curvine_block_path_pin.proto", "proto", "proto2"
    st = fd.enum_type.add()
    st.name = "StorageTypeProto"
    for i, n in enumerate(["MEM", "SSD", "HDD", "UFS", "DISK", "SPDK_DISK"]):
        v = st.value.add()
        v.name, v.number = "STORAGE_TYPE_PROTO_" + n, i
    ft = fd.enum_type.add()
    ft.name = "FileTypeProto"
    for i, n in enumerate(["DIR", "FILE", "LINK", "STREAM", "AGG", "OBJECT"]):
        v = ft.value.add()
        v.name, v.number = "FILE_TYPE_PROTO_" + n, i

    m = fd.message_type.add()
    m.name = "ExtendedBlockProto"
    _field(m, "id", 1, F.TYPE_INT64)
    _field(m, "block_size", 2, F.TYPE_INT64)
    _field(m, "storage_type", 3, F.TYPE_ENUM, type_name=".proto.StorageTypeProto")
    _field(m, "file_type", 4, F.TYPE_ENUM, type_name=".proto.FileTypeProto")

    m = fd.message_type.add()
    m.name = "BlockWriteRequest"
    _field(m, "block", 1, F.TYPE_MESSAGE, type_name=".proto.ExtendedBlockProto")
    _field(m, "off", 2, F.TYPE_INT64)
    _field(m, "block_size", 3, F.TYPE_INT64)
    _field(m, "short_circuit", 4, F.TYPE_BOOL, default="false")
    _field(m, "client_name", 5, F.TYPE_STRING, default="")
    _field(m, "chunk_size", 6, F.TYPE_INT32)

    m = fd.message_type.add()
    m.name = "BlockWriteResponse"
    _field(m, "id", 1, F.TYPE_INT64)
    _field(m, "path", 2, F.TYPE_STRING, label=OPT)
    _field(m, "off", 3, F.TYPE_INT64)
    _field(m, "block_size", 4, F.TYPE_INT64)
    _field(m, "storage_type", 5, F.TYPE_ENUM, type_name=".proto.StorageTypeProto")

    m = fd.message_type.add()
    m.name = "BlockReadRequest"
    _field(m, "id", 1, F.TYPE_INT64)
    _field(m, "off", 2, F.TYPE_INT64)
    _field(m, "len", 3, F.TYPE_INT64)
    _field(m, "chunk_size", 4, F.TYPE_INT32)
    _field(m, "short_circuit", 5, F.TYPE_BOOL, default="false")
    _field(m, "enable_read_ahead", 8, F.TYPE_BOOL, default="true")
    _field(m, "read_ahead_len", 9, F.TYPE_INT64, default="4194304")
    _field(m, "drop_cache_len", 10, F.TYPE_INT64, default="1048576")

    m = fd.message_type.add()
    m.name = "BlockReadResponse"
    _field(m, "id", 1, F.TYPE_INT64)
    _field(m, "len", 2, F.TYPE_INT64)
    _field(m, "path", 3, F.TYPE_STRING, label=OPT)
    _field(m, "storage_type", 4, F.TYPE_ENUM, type_name=".proto.StorageTypeProto")

    m = fd.message_type.add()
    m.name = "DataHeaderProto"
    _field(m, "offset", 1, F.TYPE_INT64)
    _field(m, "flush", 2, F.TYPE_BOOL)
    _field(m, "is_last", 3, F.TYPE_BOOL)
    return fd


_pool = descriptor_pool.DescriptorPool()
_pool.Add(_file())


def cls(name):
    return message_factory.GetMessageClass(_pool.FindMessageTypeByName("proto." + name))


def build(name, **fields):
    """Message `name` with every given field SET (nested dicts for sub-messages).  A proto default of a required field is
    read back from the descriptor when the caller passes the sentinel DEFAULT."""
    m = cls(name)()
    for k, v in fields.items():
        if isinstance(v, dict):
            sub = getattr(m, k)
            for kk, vv in v.items():
                setattr(sub, kk, vv)
        else:
            if v is DEFAULT:
                v = m.DESCRIPTOR.fields_by_name[k].default_value
            setattr(m, k, v)
    assert m.IsInitialized(), "required field missing: %s" % m.FindInitializationErrors()
    return m


class _Default:
    pass


DEFAULT = _Default()


def encode(name, **fields) -> bytes:
    return build(name, **fields).SerializeToString(deterministic=True)


def decode(name, data: bytes):
    m = cls(name)()
    m.ParseFromString(data)
    return m
