"""A reader and writer for the subset of the ONNX file format (protobuf wire format) that the face-analysis models use,
with no dependency on the `onnx` package: ModelProto, GraphProto, NodeProto, AttributeProto, TensorProto and
ValueInfoProto.  Initializers as raw_data or float_data / int32_data / int64_data / double_data; attributes of type
float, int, string, tensor, floats and ints; input shapes with numeric or symbolic dimensions.  Anything else that
carries meaning (external data, sparse initializers, sub-graphs, unknown element types) raises ValueError naming the
field, instead of being skipped."""
import struct
from dataclasses import dataclass, field

import numpy as np

# TensorProto.DataType -> numpy
DTYPES = {1: np.float32, 2: np.uint8, 3: np.int8, 5: np.int16, 6: np.int32, 7: np.int64, 9: np.bool_, 10: np.float16,
          11: np.float64}
_DTYPE_IDS = {np.dtype(v): k for k, v in DTYPES.items()}
# AttributeProto.AttributeType
A_FLOAT, A_INT, A_STRING, A_TENSOR, A_GRAPH, A_FLOATS, A_INTS, A_STRINGS = 1, 2, 3, 4, 5, 6, 7, 8


@dataclass
class ValueInfo:
    name: str
    elem_type: int = 1
    shape: list = None      # ints (known) and strs (symbolic); None when the shape is not given


@dataclass
class Node:
    op_type: str
    inputs: list
    outputs: list
    name: str = ""
    attrs: dict = field(default_factory=dict)
    domain: str = ""


@dataclass
class Graph:
    nodes: list
    initializers: dict       # name -> np.ndarray
    inputs: list             # ValueInfo (initializers may also be listed, as older exporters do)
    outputs: list
    name: str = "graph"


@dataclass
class Model:
    graph: Graph
    opset: int = 13
    ir_version: int = 7
    producer: str = ""


# ------------------------------------------------------------------------------------------------------ wire format
def _varint(buf, i):
    r = shift = 0
    while True:
        b = buf[i]
        i += 1
        r |= (b & 0x7F) << shift
        if b < 0x80:
            return r, i
        shift += 7


def _fields(buf):
    """Yields (field number, wire type, value) of one message; length-delimited values as memoryviews."""
    i, n = 0, len(buf)
    while i < n:
        key, i = _varint(buf, i)
        fno, wt = key >> 3, key & 7
        if wt == 0:
            v, i = _varint(buf, i)
        elif wt == 1:
            v, i = bytes(buf[i:i + 8]), i + 8
        elif wt == 2:
            ln, i = _varint(buf, i)
            v, i = buf[i:i + ln], i + ln
        elif wt == 5:
            v, i = bytes(buf[i:i + 4]), i + 4
        else:
            raise ValueError(f"unsupported protobuf wire type {wt} (field {fno})")
        if i > n:
            raise ValueError("truncated protobuf message")
        yield fno, wt, v


def _signed(v):
    return v - (1 << 64) if v >= 1 << 63 else v


def _ints(wt, v, out):
    """A repeated int64 / int32 field, packed or not."""
    if wt == 0:
        out.append(_signed(v))
    else:
        j = 0
        while j < len(v):
            x, j = _varint(v, j)
            out.append(_signed(x))


def _floats(wt, v, out, fmt="<f", size=4):
    if wt == 2:
        out.extend(struct.unpack(f"<{len(v) // size}{fmt[1]}", bytes(v)))
    else:
        out.append(struct.unpack(fmt, v)[0])


def _str(v):
    return bytes(v).decode("utf-8")


def parse_tensor(buf, where="tensor"):
    dims, dtype, raw, name = [], 1, None, ""
    data = {4: [], 5: [], 7: [], 10: []}
    for fno, wt, v in _fields(buf):
        if fno == 1:
            _ints(wt, v, dims)
        elif fno == 2:
            dtype = v
        elif fno == 8:
            name = _str(v)
        elif fno == 9:
            raw = bytes(v)
        elif fno == 4:
            _floats(wt, v, data[4])
        elif fno == 10:
            _floats(wt, v, data[10], "<d", 8)
        elif fno in (5, 7):
            _ints(wt, v, data[fno])
        elif fno == 13:
            raise ValueError(f"{where} {name!r}: external_data is not supported (save the model with its weights inside)")
        elif fno == 14:
            if v != 0:
                raise ValueError(f"{where} {name!r}: data_location={v} (external) is not supported")
        elif fno in (6, 11):
            raise ValueError(f"{where} {name!r}: field {'string_data' if fno == 6 else 'uint64_data'} is not supported")
        elif fno == 3:
            raise ValueError(f"{where} {name!r}: segmented tensors are not supported")
    if dtype not in DTYPES:
        raise ValueError(f"{where} {name!r}: data_type {dtype} is not supported")
    npt = np.dtype(DTYPES[dtype])
    count = int(np.prod(dims)) if dims else 1
    if raw is not None:
        arr = np.frombuffer(raw, dtype=npt.newbyteorder("<")).astype(npt)
    elif dtype in (1, 11):
        arr = np.array(data[4] if dtype == 1 else data[10], dtype=npt)
    elif dtype == 7:
        arr = np.array(data[7], dtype=npt)
    elif dtype == 10:   # float16 in int32_data holds the bit patterns
        arr = np.array(data[5], dtype=np.uint16).view(np.float16)
    else:
        arr = np.array(data[5], dtype=npt)
    if arr.size != count:
        raise ValueError(f"{where} {name!r}: {arr.size} values for dims {dims}")
    return name, arr.reshape(dims)


def _parse_attr(buf, node):
    name, atype, val = "", 0, None
    fl, it, ts = [], [], []
    for fno, wt, v in _fields(buf):
        if fno == 1:
            name = _str(v)
        elif fno == 20:
            atype = v
        elif fno == 2:
            val = struct.unpack("<f", v)[0]
        elif fno == 3:
            val = _signed(v)
        elif fno == 4:
            val = bytes(v)
        elif fno == 5:
            val = parse_tensor(v, f"node {node!r} attribute tensor")[1]
        elif fno == 7:
            _floats(wt, v, fl)
        elif fno == 8:
            _ints(wt, v, it)
        elif fno in (6, 9, 10, 11, 22, 21):
            raise ValueError(f"node {node!r}: attribute field {fno} (graphs, strings, tensors, sparse or referenced "
                             "attributes) is not supported")
    if atype == A_FLOATS:
        val = fl
    elif atype == A_INTS:
        val = it
    elif atype not in (A_FLOAT, A_INT, A_STRING, A_TENSOR):
        raise ValueError(f"node {node!r}: attribute {name!r} has unsupported type {atype}")
    return name, val


def _parse_node(buf):
    ins, outs, name, op, dom, attr_bufs = [], [], "", "", "", []
    for fno, wt, v in _fields(buf):
        if fno == 1:
            ins.append(_str(v))
        elif fno == 2:
            outs.append(_str(v))
        elif fno == 3:
            name = _str(v)
        elif fno == 4:
            op = _str(v)
        elif fno == 7:
            dom = _str(v)
        elif fno == 5:
            attr_bufs.append(v)
    n = Node(op, ins, outs, name, {}, dom)
    for ab in attr_bufs:
        k, val = _parse_attr(ab, name or op)
        n.attrs[k] = val
    return n


def _parse_value_info(buf):
    name, elem, shape = "", 1, None
    for fno, wt, v in _fields(buf):
        if fno == 1:
            name = _str(v)
        elif fno == 2:
            for f2, _, tt in _fields(v):
                if f2 != 1:
                    raise ValueError(f"value {name!r}: only tensor types are supported")
                for f3, _, tv in _fields(tt):
                    if f3 == 1:
                        elem = tv
                    elif f3 == 2:
                        shape = []
                        for f4, _, dv in _fields(tv):
                            if f4 != 1:
                                continue
                            d = "?"
                            for f5, _, x in _fields(dv):
                                if f5 == 1:
                                    d = _signed(x)
                                elif f5 == 2:
                                    d = _str(x)
                            shape.append(d)
    return ValueInfo(name, elem, shape)


def _parse_graph(buf):
    g = Graph([], {}, [], [])
    for fno, wt, v in _fields(buf):
        if fno == 1:
            g.nodes.append(_parse_node(v))
        elif fno == 2:
            g.name = _str(v)
        elif fno == 5:
            k, arr = parse_tensor(v, "initializer")
            g.initializers[k] = arr
        elif fno == 15:
            raise ValueError("graph: sparse_initializer is not supported")
        elif fno == 11:
            g.inputs.append(_parse_value_info(v))
        elif fno == 12:
            g.outputs.append(_parse_value_info(v))
    return g


def loads(data: bytes) -> Model:
    buf = memoryview(data)
    graph, opset, ir, prod = None, None, 0, ""
    for fno, wt, v in _fields(buf):
        if fno == 1:
            ir = v
        elif fno == 2:
            prod = _str(v)
        elif fno == 7:
            graph = _parse_graph(v)
        elif fno == 8:
            dom, ver = "", 0
            for f2, _, x in _fields(v):
                if f2 == 1:
                    dom = _str(x)
                elif f2 == 2:
                    ver = x
            if dom in ("", "ai.onnx"):
                opset = ver
        elif fno == 25:
            raise ValueError("model: local functions are not supported")
    if graph is None:
        raise ValueError("model: no graph (not an ONNX model file?)")
    return Model(graph, opset or 1, ir, prod)


def load(path) -> Model:
    with open(path, "rb") as f:
        return loads(f.read())


# ------------------------------------------------------------------------------------------------------------ writer
def _wvarint(n):
    if n < 0:
        n += 1 << 64
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _key(fno, wt):
    return _wvarint((fno << 3) | wt)


def _wint(fno, v):
    return _key(fno, 0) + _wvarint(int(v))


def _wbytes(fno, b):
    return _key(fno, 2) + _wvarint(len(b)) + b


def _wstr(fno, s):
    return _wbytes(fno, s.encode("utf-8"))


def _wpacked_ints(fno, vals):
    return _wbytes(fno, b"".join(_wvarint(int(v)) for v in vals)) if len(vals) else b""


def dump_tensor(name, arr):
    arr = np.asarray(arr)
    if arr.dtype not in _DTYPE_IDS:
        raise ValueError(f"tensor {name!r}: numpy type {arr.dtype} has no ONNX data type here")
    b = _wpacked_ints(1, arr.shape) + _wint(2, _DTYPE_IDS[arr.dtype]) + _wstr(8, name)
    return b + _wbytes(9, np.ascontiguousarray(arr).astype(arr.dtype.newbyteorder("<")).tobytes())


def _dump_attr(name, val):
    b = _wstr(1, name)
    if isinstance(val, bool) or isinstance(val, (int, np.integer)):
        return b + _wint(20, A_INT) + _wint(3, val)
    if isinstance(val, float):
        return b + _wint(20, A_FLOAT) + _key(2, 5) + struct.pack("<f", val)
    if isinstance(val, (bytes, str)):
        return b + _wint(20, A_STRING) + _wbytes(4, val.encode() if isinstance(val, str) else val)
    if isinstance(val, np.ndarray):
        return b + _wint(20, A_TENSOR) + _wbytes(5, dump_tensor("", val))
    if isinstance(val, (list, tuple)) and all(isinstance(x, (int, np.integer)) for x in val):
        return b + _wint(20, A_INTS) + _wpacked_ints(8, val)
    if isinstance(val, (list, tuple)):
        return b + _wint(20, A_FLOATS) + _wbytes(7, struct.pack(f"<{len(val)}f", *val))
    raise ValueError(f"attribute {name!r}: cannot encode {type(val).__name__}")


def _dump_value_info(vi):
    t = _wint(1, vi.elem_type)
    if vi.shape is not None:
        dims = b"".join(_wbytes(1, _wstr(2, d) if isinstance(d, str) else _wint(1, d)) for d in vi.shape)
        t += _wbytes(2, dims)
    return _wstr(1, vi.name) + _wbytes(2, _wbytes(1, t))


def dumps(model: Model) -> bytes:
    g = model.graph
    gb = b""
    for n in g.nodes:
        nb = b"".join(_wstr(1, x) for x in n.inputs) + b"".join(_wstr(2, x) for x in n.outputs)
        nb += _wstr(3, n.name) + _wstr(4, n.op_type) + (_wstr(7, n.domain) if n.domain else b"")
        nb += b"".join(_wbytes(5, _dump_attr(k, v)) for k, v in n.attrs.items())
        gb += _wbytes(1, nb)
    gb += _wstr(2, g.name)
    gb += b"".join(_wbytes(5, dump_tensor(k, v)) for k, v in g.initializers.items())
    gb += b"".join(_wbytes(11, _dump_value_info(v)) for v in g.inputs)
    gb += b"".join(_wbytes(12, _dump_value_info(v)) for v in g.outputs)
    opset = _wbytes(8, _wstr(1, "") + _wint(2, model.opset))
    return _wint(1, model.ir_version) + _wstr(2, model.producer) + _wbytes(7, gb) + opset


def save(model: Model, path):
    with open(path, "wb") as f:
        f.write(dumps(model))
