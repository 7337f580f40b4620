"""Pinot immutable-segment writer (tooling, CPU).

Emits the exact per-column index buffers a Pinot v3 segment holds, so that the
synthetic-table generator and the test fixtures can feed the GPU executor (and
the oracle) the same bytes `ImmutableSegmentLoader` would mmap.  Only the index
types on the hot path are written: dictionary, fixed-bit / sorted / raw forward
index, bitmap inverted index.

Layouts follow (restated, not copied):
  dictionary         SEGL/segment/index/readers/BaseImmutableDictionary.java:45-58,
                     SEGL/io/util/FixedByteValueReaderWriter.java:36-54 (big-endian, sorted)
  bits per element   SEGL/io/util/PinotDataBitSet.java:61-72
  unsorted fwd       SEGL/io/writer/impl/FixedBitSVForwardIndexWriter.java:40-46
  sorted fwd         SEGL/segment/index/readers/sorted/SortedIndexReaderImpl.java:37-41,114-116
  raw fwd (v2)       SEGL/io/writer/impl/BaseChunkForwardIndexWriter.java:40-60,120-160
  inverted           SEGL/segment/creator/impl/inv/BitmapInvertedIndexWriter.java:35-50
  v3 directory       SEGL/segment/store/SingleFileIndexDirectory.java:72-73,174-204
(SEGL = pinot-segment-local/src/main/java/org/apache/pinot/segment/local)
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from collections import OrderedDict
from dataclasses import dataclass, field
from enum import IntEnum
from typing import Dict, List, Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SEGW_SO = os.path.join(_HERE, "libpinot_b200_segwriter.so")
_SEGW_SRC = os.path.join(_HERE, "csrc", "segment_writer.c")


class DataType(IntEnum):
    INT = 0
    LONG = 1
    FLOAT = 2
    DOUBLE = 3
    STRING = 4


_NP_BE = {DataType.INT: ">i4", DataType.LONG: ">i8", DataType.FLOAT: ">f4", DataType.DOUBLE: ">f8"}
_NP_NATIVE = {DataType.INT: np.int32, DataType.LONG: np.int64, DataType.FLOAT: np.float32,
              DataType.DOUBLE: np.float64}
_WIDTH = {DataType.INT: 4, DataType.LONG: 8, DataType.FLOAT: 4, DataType.DOUBLE: 8}

RAW_DOCS_PER_CHUNK = 1000        # ForwardIndexConfig default targetDocsPerChunk
RAW_WRITER_VERSION = 2           # ForwardIndexConfig.DEFAULT_RAW_WRITER_VERSION
COMPRESSION_PASS_THROUGH = 0     # ChunkCompressionType.PASS_THROUGH
MAGIC_MARKER = 0xDEADBEEFDEAFBEAD


def build_segwriter(force: bool = False) -> str:
    """Compile the C helper in-tree (gcc only, no CUDA)."""
    if force or not os.path.exists(_SEGW_SO) or os.path.getmtime(_SEGW_SO) < os.path.getmtime(_SEGW_SRC):
        subprocess.check_call(["gcc", "-O3", "-shared", "-fPIC", "-o", _SEGW_SO, _SEGW_SRC])
    return _SEGW_SO


_lib = None


def _segw():
    global _lib
    if _lib is None:
        lib = ctypes.CDLL(build_segwriter())
        lib.pbw_pack_bits_be.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
        lib.pbw_pack_bits_be.restype = None
        lib.pbw_unpack_bits_be.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
        lib.pbw_unpack_bits_be.restype = None
        lib.pbw_roaring_serialize.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_void_p,
                                              ctypes.c_int64]
        lib.pbw_roaring_serialize.restype = ctypes.c_int64
        lib.pbw_build_inverted_index.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_int,
                                                 ctypes.c_void_p, ctypes.c_int64]
        lib.pbw_build_inverted_index.restype = ctypes.c_int64
        _lib = lib
    return _lib


def num_bits_per_value(max_value: int) -> int:
    """PinotDataBitSet.getNumBitsPerValue: at least 1 bit."""
    if max_value <= 1:
        return 1
    return int(max_value).bit_length()


def pack_bits_be(values: np.ndarray, w: int) -> np.ndarray:
    v = np.ascontiguousarray(values, dtype=np.uint32)
    out = np.zeros((v.size * w + 7) // 8, dtype=np.uint8)
    _segw().pbw_pack_bits_be(v.ctypes.data, v.size, w, out.ctypes.data)
    return out


def unpack_bits_be(buf: np.ndarray, n: int, w: int) -> np.ndarray:
    b = np.ascontiguousarray(buf, dtype=np.uint8)
    out = np.empty(n, dtype=np.uint32)
    _segw().pbw_unpack_bits_be(b.ctypes.data, n, w, out.ctypes.data)
    return out


def roaring_serialize(doc_ids: np.ndarray, run_optimize: bool = True) -> np.ndarray:
    d = np.ascontiguousarray(doc_ids, dtype=np.uint32)
    need = _segw().pbw_roaring_serialize(d.ctypes.data, d.size, int(run_optimize), None, 0)
    if need < 0:
        raise ValueError("roaring serialise failed")
    out = np.zeros(need, dtype=np.uint8)
    got = _segw().pbw_roaring_serialize(d.ctypes.data, d.size, int(run_optimize), out.ctypes.data, need)
    assert got == need
    return out


def build_inverted_index(dict_ids: np.ndarray, card: int, run_optimize: bool = True) -> np.ndarray:
    d = np.ascontiguousarray(dict_ids, dtype=np.uint32)
    need = _segw().pbw_build_inverted_index(d.ctypes.data, d.size, card, int(run_optimize), None, 0)
    if need < 0:
        raise ValueError("inverted index build failed")
    out = np.zeros(need, dtype=np.uint8)
    got = _segw().pbw_build_inverted_index(d.ctypes.data, d.size, card, int(run_optimize), out.ctypes.data, need)
    assert got == need
    return out


@dataclass
class ColumnIndex:
    """One column's index buffers exactly as they sit in columns.psf."""
    name: str
    data_type: DataType
    num_docs: int
    has_dictionary: bool
    is_sorted: bool
    cardinality: int
    bits_per_element: int
    dict_entry_bytes: int                    # lengthOfEachEntry
    forward_index: np.ndarray                # uint8
    dictionary: Optional[np.ndarray] = None  # uint8
    inverted_index: Optional[np.ndarray] = None
    null_value_vector: Optional[np.ndarray] = None   # <col>.bitmap.nullvalue: RoaringBitmap of the null docIds (absent when none)
    min_value: object = None
    max_value: object = None

    @property
    def fwd_kind(self) -> str:
        if not self.has_dictionary:
            return "raw"
        return "sorted" if self.is_sorted else "unsorted"

    def dictionary_values(self) -> np.ndarray:
        """Decoded dictionary (native numpy array; bytes objects for STRING)."""
        assert self.has_dictionary
        if self.data_type == DataType.STRING and is_var_length_dictionary(self.dictionary):
            d = self.dictionary
            data0 = int(d[12:16].view(">i4")[0])
            offs = d[data0:data0 + 4 * (self.cardinality + 1)].view(">i4").astype(np.int64)
            return np.array([bytes(d[offs[i]:offs[i + 1]]) for i in range(self.cardinality)], dtype=object)
        if self.data_type == DataType.STRING:
            raw = self.dictionary.reshape(self.cardinality, self.dict_entry_bytes)
            return np.array([bytes(r).rstrip(b"\0") for r in raw], dtype=object)
        return self.dictionary.view(_NP_BE[self.data_type]).astype(_NP_NATIVE[self.data_type])


@dataclass
class Segment:
    name: str
    num_docs: int
    columns: "OrderedDict[str, ColumnIndex]" = field(default_factory=OrderedDict)

    def column_names(self) -> List[str]:
        return list(self.columns.keys())


VAR_LENGTH_MAGIC = b".vl;"


def _encode_var_length_dictionary(values_sorted) -> np.ndarray:
    """VarLengthValueWriter (SEGL/io/util/VarLengthValueWriter.java:78-125): magic, version 1, numValues,
    dataSectionStartOffset (= header length 16), numValues + 1 big-endian int offsets from the buffer start, the bytes."""
    n = len(values_sorted)
    off0 = 16 + 4 * (n + 1)
    lens = np.array([len(v) for v in values_sorted], dtype=np.int64)
    offs = off0 + np.concatenate([[0], np.cumsum(lens)])
    head = VAR_LENGTH_MAGIC + np.array([1, n, 16], dtype=">i4").tobytes() + offs.astype(">i4").tobytes()
    return np.frombuffer(head + b"".join(bytes(v) for v in values_sorted), dtype=np.uint8).copy()


def is_var_length_dictionary(buf: np.ndarray) -> bool:
    return buf is not None and buf.size >= 20 and bytes(buf[:4]) == VAR_LENGTH_MAGIC and int(buf[4:8].view(">i4")[0]) == 1


def _encode_dictionary(values_sorted: np.ndarray, data_type: DataType, var_length: bool = False):
    if data_type == DataType.STRING and var_length:
        return _encode_var_length_dictionary(values_sorted), max(1, max(len(v) for v in values_sorted))
    if data_type == DataType.STRING:
        width = max(1, max(len(v) for v in values_sorted))
        buf = np.zeros((len(values_sorted), width), dtype=np.uint8)
        for i, v in enumerate(values_sorted):
            buf[i, :len(v)] = np.frombuffer(v, dtype=np.uint8)
        return buf.reshape(-1), width
    be = np.asarray(values_sorted).astype(_NP_BE[data_type])
    return np.frombuffer(be.tobytes(), dtype=np.uint8).copy(), _WIDTH[data_type]


def _sorted_pairs(dict_ids: np.ndarray, card: int) -> np.ndarray:
    """(startDocId, endDocId) inclusive per dictId, big-endian int32."""
    n = dict_ids.size
    starts = np.searchsorted(dict_ids, np.arange(card), side="left")
    ends = np.searchsorted(dict_ids, np.arange(card), side="right") - 1
    assert n == 0 or (ends >= starts).all(), "every dictId must occur in a sorted column"
    pairs = np.stack([starts, ends], axis=1).astype(">i4")
    return np.frombuffer(pairs.tobytes(), dtype=np.uint8).copy()


COMPRESSION_SNAPPY = 1           # ChunkCompressionType ordinals (SPI/compression/ChunkCompressionType.java:22)
COMPRESSION_LZ4 = 3
COMPRESSION_LZ4_LENGTH_PREFIXED = 4
_COMPRESSION_BY_NAME = {None: 0, "PASS_THROUGH": 0, "SNAPPY": 1, "LZ4": 3, "LZ4_LENGTH_PREFIXED": 4}


def _compress_chunk(raw: bytes, compression: int, block=None) -> bytes:
    """One chunk through the codec Pinot's ChunkCompressorFactory would use.  The compressors are pyarrow's bindings of the
    stock C libraries (liblz4 block format = lz4-java's fastCompressor output format; raw snappy = snappy-java's): this
    module only frames them the way the reference's writers do.  block: raw chunk -> LZ4 block or Snappy stream, in place
    of the stock compressor (tests that emit chosen stream features)."""
    import pyarrow as pa
    if block is not None:
        z = block(raw)
    elif compression == COMPRESSION_SNAPPY:
        return pa.Codec("snappy").compress(raw, asbytes=True)
    else:
        z = pa.Codec("lz4_raw").compress(raw, asbytes=True)
    if compression == COMPRESSION_LZ4_LENGTH_PREFIXED:        # lz4-java LZ4CompressorWithLength: little-endian decoded length
        return len(raw).to_bytes(4, "little") + z
    return z


def _raw_forward_index(values: np.ndarray, data_type: DataType, compression=None, version: int = RAW_WRITER_VERSION,
                       docs_per_chunk: int = RAW_DOCS_PER_CHUNK, block=None) -> np.ndarray:
    """BaseChunkForwardIndexWriter / FixedByteChunkForwardIndexWriter (SEGL/io/writer/impl/BaseChunkForwardIndexWriter.java:
    73-190): header of seven big-endian ints (version, numChunks, numDocsPerChunk, sizeOfEntry, totalDocs, compressionType,
    dataHeaderStart), chunk offsets (int for versions 1 and 2, long for 3 and 4), then the chunks, each compressed on its
    own; the last chunk holds only the docs that are left.  Version 1 has only the first four header ints and no
    compression field: its chunks are always SNAPPY.  block: see _compress_chunk."""
    comp = _COMPRESSION_BY_NAME[compression] if not isinstance(compression, int) else compression
    assert version in (1, 2, 3, 4)
    assert version > 1 or comp == COMPRESSION_SNAPPY, "version 1 chunks are SNAPPY"
    n = values.size
    width = _WIDTH[data_type]
    num_chunks = (n + docs_per_chunk - 1) // docs_per_chunk
    off_dtype = ">i4" if version <= 2 else ">i8"
    n_header_ints = 4 if version == 1 else 7
    header_size = n_header_ints * 4 + num_chunks * (4 if version <= 2 else 8)
    header = np.empty(7, dtype=">i4")
    header[0] = version
    header[1] = num_chunks
    header[2] = docs_per_chunk
    header[3] = width
    header[4] = n
    header[5] = comp
    header[6] = 7 * 4                              # dataHeaderStart
    header = header[:n_header_ints]
    body = np.asarray(values).astype(_NP_BE[data_type]).tobytes()
    if comp == 0:
        offs = header_size + np.arange(num_chunks, dtype=np.int64) * (docs_per_chunk * width)
        chunks = [body]
    else:
        chunks, offs, pos = [], [], header_size
        step = docs_per_chunk * width
        for k in range(num_chunks):
            z = _compress_chunk(body[k * step:(k + 1) * step], comp, block)
            offs.append(pos)
            chunks.append(z)
            pos += len(z)
        offs = np.asarray(offs, dtype=np.int64)
    return np.frombuffer(header.tobytes() + offs.astype(off_dtype).tobytes() + b"".join(chunks), dtype=np.uint8).copy()


def java_string_key(b: bytes) -> bytes:
    """Sort key that orders UTF-8 byte strings like java.lang.String.compareTo (by UTF-16 code units)."""
    try:
        return b.decode("utf-8").encode("utf-16-be", "surrogatepass")
    except UnicodeDecodeError:
        return b


def build_dict_column(name: str, data_type: DataType, dict_values_sorted: np.ndarray, dict_ids: np.ndarray,
                      inverted: bool = False, run_optimize: bool = True, var_length_dictionary: bool = False) -> ColumnIndex:
    """Column from an already-known sorted dictionary and per-doc dictIds."""
    card = len(dict_values_sorted)
    dict_ids = np.ascontiguousarray(dict_ids, dtype=np.uint32)
    n = dict_ids.size
    bits = num_bits_per_value(card - 1)
    dbuf, width = _encode_dictionary(dict_values_sorted, data_type, var_length_dictionary)
    is_sorted = bool(n <= 1 or (dict_ids[1:] >= dict_ids[:-1]).all())
    fwd = _sorted_pairs(dict_ids, card) if is_sorted else pack_bits_be(dict_ids, bits)
    inv = build_inverted_index(dict_ids, card, run_optimize) if (inverted and not is_sorted) else None
    return ColumnIndex(name=name, data_type=data_type, num_docs=n, has_dictionary=True, is_sorted=is_sorted,
                       cardinality=card, bits_per_element=bits, dict_entry_bytes=width, forward_index=fwd,
                       dictionary=dbuf, inverted_index=inv, min_value=dict_values_sorted[0],
                       max_value=dict_values_sorted[-1])


def build_column(name: str, data_type: DataType, values, dictionary: bool = True, inverted: bool = False,
                 run_optimize: bool = True, var_length_dictionary: bool = False, raw_compression=None,
                 raw_version: int = RAW_WRITER_VERSION, raw_docs_per_chunk: int = RAW_DOCS_PER_CHUNK, raw_block=None) -> ColumnIndex:
    """Column from per-doc values (what SegmentIndexCreationDriverImpl does per column).  raw_block: see _compress_chunk."""
    if data_type == DataType.STRING:
        vals = np.array([v if isinstance(v, bytes) else str(v).encode("utf-8") for v in values], dtype=object)
        assert dictionary, "raw STRING columns are out of scope"
        # the dictionary is sorted by String.compareTo = UTF-16 code units (SegmentDictionaryCreator sorts the Java strings);
        # for anything below U+10000 that is the byte order of the UTF-8 encodings as well
        uniq_b, inv_ids = np.unique(vals, return_inverse=True)
        order = sorted(range(len(uniq_b)), key=lambda i: java_string_key(uniq_b[i]))
        rank = np.empty(len(order), dtype=np.int64)
        rank[np.asarray(order, dtype=np.int64)] = np.arange(len(order))
        uniq = np.array([uniq_b[i] for i in order], dtype=object)
        return build_dict_column(name, data_type, uniq, rank[inv_ids].astype(np.uint32), inverted, run_optimize, var_length_dictionary)
    vals = np.asarray(values).astype(_NP_NATIVE[data_type])
    if dictionary:
        uniq, inv_ids = np.unique(vals, return_inverse=True)
        return build_dict_column(name, data_type, uniq, inv_ids.astype(np.uint32), inverted, run_optimize)
    n = vals.size
    is_sorted = bool(n <= 1 or (vals[1:] >= vals[:-1]).all())
    return ColumnIndex(name=name, data_type=data_type, num_docs=n, has_dictionary=False, is_sorted=is_sorted,
                       cardinality=-1, bits_per_element=-1, dict_entry_bytes=_WIDTH[data_type],
                       forward_index=_raw_forward_index(vals, data_type, raw_compression, raw_version, raw_docs_per_chunk, raw_block),
                       min_value=vals.min() if n else None, max_value=vals.max() if n else None)


def with_nulls(col: ColumnIndex, null_mask) -> ColumnIndex:
    """Attach a null-value vector (NullValueVectorCreator: SEGL/segment/creator/impl/nullvalue/NullValueVectorCreator.java --
    one run-compressed RoaringBitmap of the docIds whose value was null; the forward index holds the column's default null
    value at those docs, which is the caller's business; no file when nothing is null)."""
    docs = np.flatnonzero(np.asarray(null_mask, dtype=bool)).astype(np.uint32)
    assert np.asarray(null_mask).size == col.num_docs
    col.null_value_vector = roaring_serialize(docs, run_optimize=True) if docs.size else None
    return col


def make_segment(name: str, columns: List[ColumnIndex]) -> Segment:
    n = columns[0].num_docs
    assert all(c.num_docs == n for c in columns)
    seg = Segment(name=name, num_docs=n)
    for c in columns:
        seg.columns[c.name] = c
    return seg


# ----------------------------------------------------------------------------
# v3 directory (columns.psf + index_map + metadata.properties)
# ----------------------------------------------------------------------------

def write_v3(seg: Segment, out_dir: str, table_name: str = "testTable") -> str:
    v3 = os.path.join(out_dir, seg.name, "v3")
    os.makedirs(v3, exist_ok=True)
    index_map: List[str] = []
    magic = MAGIC_MARKER.to_bytes(8, "big")
    with open(os.path.join(v3, "columns.psf"), "wb") as f:
        off = 0
        for c in seg.columns.values():
            parts = []
            if c.dictionary is not None:
                parts.append(("dictionary", c.dictionary))
            parts.append(("forward_index", c.forward_index))
            if c.inverted_index is not None:
                parts.append(("inverted_index", c.inverted_index))
            if c.null_value_vector is not None:
                parts.append(("nullvalue_vector", c.null_value_vector))     # StandardIndexes.nullValueVector() id
            for kind, buf in parts:
                f.write(magic)
                f.write(buf.tobytes())
                size = 8 + buf.size
                index_map.append(f"{c.name}.{kind}.startOffset = {off}")
                index_map.append(f"{c.name}.{kind}.size = {size}")
                off += size
    with open(os.path.join(v3, "index_map"), "w") as f:
        f.write("\n".join(index_map) + "\n")
    md = [f"segment.name = {seg.name}", f"segment.table.name = {table_name}",
          f"segment.total.docs = {seg.num_docs}", "segment.index.version = v3",
          "segment.dimension.column.names = " + ",".join(seg.columns.keys())]
    for c in seg.columns.values():
        p = f"column.{c.name}."
        md += [p + f"cardinality = {c.cardinality}", p + f"totalDocs = {c.num_docs}",
               p + f"dataType = {c.data_type.name}", p + f"bitsPerElement = {c.bits_per_element}",
               p + f"lengthOfEachEntry = {c.dict_entry_bytes if c.data_type == DataType.STRING else 0}",
               p + f"isSorted = {str(c.is_sorted).lower()}", p + f"hasDictionary = {str(c.has_dictionary).lower()}",
               p + "isSingleValues = true", p + "maxNumberOfMultiValues = 0",
               p + f"totalNumberOfEntries = {c.num_docs}"]
    with open(os.path.join(v3, "metadata.properties"), "w") as f:
        f.write("\n".join(md) + "\n")
    return os.path.join(out_dir, seg.name)


def load_v3(segment_dir: str) -> Segment:
    """Open a v3 segment directory the way Pinot's SingleFileIndexDirectory does (SEGL/segment/store/
    SingleFileIndexDirectory.java:72-73, 174-204): `index_map` gives (startOffset, size) of every index inside
    `columns.psf`, each slice starts with the 8-byte magic marker 0xdeadbeefdeafbead, and the index buffer is the view
    after the marker.  Buffers are zero-copy read-only views of one np.memmap (like PinotDataBuffer views of the mmap'd
    file), so they sit at arbitrary byte offsets — exactly what the stager has to cope with in a server."""
    v3 = os.path.join(segment_dir, "v3")
    props: Dict[str, str] = {}
    with open(os.path.join(v3, "metadata.properties")) as f:
        for line in f:
            if "=" in line:
                k, v = line.split("=", 1)
                props[k.strip()] = v.strip()
    slices: Dict[tuple, List[int]] = {}
    with open(os.path.join(v3, "index_map")) as f:
        for line in f:
            if "=" not in line:
                continue
            k, v = (x.strip() for x in line.split("=", 1))
            col, kind, what = k.rsplit(".", 2)
            slices.setdefault((col, kind), [0, 0])[0 if what == "startOffset" else 1] = int(v)
    psf = np.memmap(os.path.join(v3, "columns.psf"), dtype=np.uint8, mode="r")
    magic = np.frombuffer(MAGIC_MARKER.to_bytes(8, "big"), dtype=np.uint8)

    def view(col: str, kind: str) -> Optional[np.ndarray]:
        if (col, kind) not in slices:
            return None
        off, size = slices[(col, kind)]
        if not (psf[off:off + 8] == magic).all():
            raise ValueError(f"{col}.{kind}: magic marker missing at offset {off}")
        return psf[off + 8:off + size]

    seg = Segment(props["segment.name"], int(props["segment.total.docs"]))
    for name in props["segment.dimension.column.names"].split(","):
        p = f"column.{name}."
        dt = DataType[props[p + "dataType"]]
        has_dict = props[p + "hasDictionary"] == "true"
        width = int(props[p + "lengthOfEachEntry"]) if dt == DataType.STRING else _WIDTH[dt]
        seg.columns[name] = ColumnIndex(
            name=name, data_type=dt, num_docs=int(props[p + "totalDocs"]), has_dictionary=has_dict,
            is_sorted=props[p + "isSorted"] == "true", cardinality=int(props[p + "cardinality"]),
            bits_per_element=int(props[p + "bitsPerElement"]), dict_entry_bytes=width,
            forward_index=view(name, "forward_index"), dictionary=view(name, "dictionary") if has_dict else None,
            inverted_index=view(name, "inverted_index"), null_value_vector=view(name, "nullvalue_vector"))
    return seg
