"""Pinot on-disk layouts: the tooling writer against the oracle's reader and against independent numpy / Python decoders.
Mirrors the property tests of the reference (PinotDataBitSetTest, FixedBitIntReaderTest, BitmapInvertedIndex*Test) — those
hold no literal vectors — plus the structure of the RoaringBitmap portable format.  CPU only."""
import ctypes as C
import struct

import numpy as np
import pytest

from oracle import oracle
from pinot_b200.segment_writer import (DataType, build_column, build_dict_column, build_inverted_index, num_bits_per_value,
                                       pack_bits_be, roaring_serialize, unpack_bits_be)


def test_num_bits_per_value():   # PinotDataBitSetTest.testGetNumBitsPerValue (PinotDataBitSet.java:61-72)
    l = oracle.lib()
    assert l.orc_num_bits_per_value(0) == 1 and num_bits_per_value(0) == 1
    rng = np.random.default_rng(1)
    for v in [1, 2, 3, 4, 255, 256, 65535, 65536, 2**31 - 1] + rng.integers(1, 2**31 - 1, 200).tolist():
        assert l.orc_num_bits_per_value(int(v)) == int(v).bit_length() == num_bits_per_value(int(v))


@pytest.mark.parametrize("w", list(range(1, 32)))
def test_fixed_bit_stream_round_trip(w):   # PinotDataBitSetTest.testReadWriteInt / FixedBitIntReaderTest: MSB-first, value i at bit i*w
    rng = np.random.default_rng(w)
    n = 1000 + w
    vals = rng.integers(0, 2**w, n, dtype=np.uint64).astype(np.uint32)
    vals[0], vals[-1] = 2**w - 1, 0
    buf = pack_bits_be(vals, w)
    assert buf.nbytes == (n * w + 7) // 8                                      # FixedBitSVForwardIndexWriter.java:40-46
    # independent decoder: the whole stream as one big-endian integer
    big = int.from_bytes(buf.tobytes(), "big")
    total = buf.nbytes * 8
    for i in (0, 1, 2, 31, 32, 33, n // 2, n - 2, n - 1):
        assert (big >> (total - (i + 1) * w)) & (2**w - 1) == int(vals[i])
    assert (unpack_bits_be(buf, n, w) == vals).all()
    l = oracle.lib()
    padded = np.concatenate([buf, np.zeros(8, np.uint8)])
    for i in (0, 1, 31, 32, 33, n // 3, n - 1):
        assert l.orc_read_dict_id(padded.ctypes.data, w, i) == int(vals[i])


def _roaring_decode_py(blob: bytes, layout=None):
    """RoaringBitmap portable format, decoded from the public spec alone (cookies 12346 / 12347).  layout: a dict that
    receives the cookie, whether the blob has the offset header, and per container (key, cardinality, kind), kind one of
    'array', 'bitmap', 'run'."""
    cookie = struct.unpack_from("<I", blob, 0)[0]
    pos = 4
    if cookie & 0xFFFF == 12347:
        n = (cookie >> 16) + 1
        run_flags = blob[pos:pos + (n + 7) // 8]
        pos += (n + 7) // 8
        has_offsets = n >= 4
    else:
        assert cookie == 12346
        n = struct.unpack_from("<I", blob, pos)[0]
        pos += 4
        run_flags = bytes((n + 7) // 8)
        has_offsets = True
    keys = [struct.unpack_from("<HH", blob, pos + 4 * i) for i in range(n)]
    pos += 4 * n
    if has_offsets:
        pos += 4 * n
    out = []
    if layout is not None:
        layout.update(cookie=cookie & 0xFFFF, offsets=has_offsets, containers=[])
    for i, (key, card_m1) in enumerate(keys):
        card = card_m1 + 1
        base = key << 16
        if layout is not None:
            kind = "run" if run_flags[i // 8] >> (i % 8) & 1 else "bitmap" if card > 4096 else "array"
            layout["containers"].append((key, card, kind))
        if run_flags[i // 8] >> (i % 8) & 1:
            nr = struct.unpack_from("<H", blob, pos)[0]
            pos += 2
            for r in range(nr):
                s, ln = struct.unpack_from("<HH", blob, pos)
                pos += 4
                out.extend(range(base + s, base + s + ln + 1))
        elif card > 4096:
            words = struct.unpack_from("<1024Q", blob, pos)
            pos += 8192
            for wi, wv in enumerate(words):
                while wv:
                    b = (wv & -wv).bit_length() - 1
                    out.append(base + wi * 64 + b)
                    wv &= wv - 1
        else:
            out.extend(base + v for v in struct.unpack_from(f"<{card}H", blob, pos))
            pos += 2 * card
    assert pos == len(blob)
    return out


@pytest.mark.parametrize("shape", ["empty", "sparse", "dense", "runs", "mixed_many_containers", "single"])
@pytest.mark.parametrize("run_optimize", [True, False])
def test_roaring_portable_format(shape, run_optimize):
    rng = np.random.default_rng(5)
    if shape == "empty":
        docs = np.zeros(0, np.uint32)
    elif shape == "single":
        docs = np.array([70000], np.uint32)
    elif shape == "sparse":
        docs = np.unique(rng.integers(0, 300_000, 900)).astype(np.uint32)                  # array containers
    elif shape == "dense":
        docs = np.unique(rng.integers(0, 131_072, 90_000)).astype(np.uint32)                # bitmap containers
    elif shape == "runs":
        docs = np.concatenate([np.arange(10, 5000), np.arange(70_000, 140_000), np.arange(200_000, 200_003)]).astype(np.uint32)
    else:
        docs = np.unique(np.concatenate([rng.integers(0, 65536 * 7, 3000), np.arange(65536 * 2 + 5, 65536 * 3 - 9),
                                         rng.integers(65536 * 4, 65536 * 5, 30_000)])).astype(np.uint32)   # >= 4 containers: offset header
    blob = roaring_serialize(docs, run_optimize)
    assert _roaring_decode_py(blob.tobytes()) == docs.tolist()
    out = np.zeros(max(docs.size, 1), np.uint32)
    n = oracle.lib().orc_roaring_to_doc_ids(blob.ctypes.data, blob.size, out.ctypes.data, out.size)
    assert n == docs.size and (out[:n] == docs).all()
    if not run_optimize and docs.size:
        assert struct.unpack_from("<I", blob.tobytes(), 0)[0] == 12346                      # no run containers without runOptimize


def test_inverted_index_buffer_layout():   # BitmapInvertedIndexWriter: (card + 1) big-endian offsets, then the bitmaps (BitmapInvertedIndexReader.java:45-62)
    rng = np.random.default_rng(9)
    card, n = 37, 50_000
    ids = rng.integers(0, card, n, dtype=np.uint32)
    ids[:card] = np.arange(card, dtype=np.uint32)
    inv = build_inverted_index(ids, card).tobytes()
    offs = struct.unpack_from(f">{card + 1}I", inv, 0)
    assert offs[0] == 4 * (card + 1) and offs[-1] == len(inv) and all(a <= b for a, b in zip(offs, offs[1:]))
    for d in (0, 1, card // 2, card - 1):
        assert _roaring_decode_py(inv[offs[d]:offs[d + 1]]) == np.nonzero(ids == d)[0].tolist()


def test_sorted_and_raw_forward_indexes():
    # sorted column: card x (startDocId, endDocId) big-endian pairs, inclusive (SortedIndexReaderImpl.java:37-116)
    ids = np.repeat(np.arange(5, dtype=np.uint32), [3, 1, 4, 2, 6])
    c = build_dict_column("s", DataType.INT, np.arange(5, dtype=np.int32) * 10, ids)
    assert c.is_sorted and struct.unpack(">10i", c.forward_index.tobytes()) == (0, 2, 3, 3, 4, 7, 8, 9, 10, 15)
    # raw PASS_THROUGH chunk index v2: 7 header ints + chunk offsets, then big-endian values (BaseChunkForwardIndexWriter / FixedByteChunkSVForwardIndexReader.java:35-61)
    vals = (np.arange(2500, dtype=np.int64) * 7919 - 5_000_000)
    r = build_column("k", DataType.LONG, vals, dictionary=False)
    raw = r.forward_index.tobytes()
    version, num_chunks, docs_per_chunk, width, total, compression, header_start = struct.unpack_from(">7i", raw, 0)
    assert (width, total, compression, header_start) == (8, 2500, 0, 28) and num_chunks == -(-2500 // docs_per_chunk)
    data0 = struct.unpack_from(">i", raw, header_start)[0]
    assert data0 == 28 + 4 * num_chunks
    assert struct.unpack_from(">3q", raw, data0) == tuple(int(v) for v in vals[:3])
    assert struct.unpack_from(">q", raw, data0 + 8 * 2499)[0] == int(vals[-1])


def test_v3_directory_round_trip(tmp_path):
    """write_v3 -> load_v3 (index_map + magic markers + one mmap'd columns.psf, SingleFileIndexDirectory.java:174-204): the
    oracle sees the same segment through views at arbitrary byte offsets of the file."""
    from pinot_b200 import datagen
    from pinot_b200.query import parse_sql
    from pinot_b200.segment_writer import load_v3, write_v3
    seg = datagen.make_segment_synth(2, 20_003, columns=["c1", "c3", "d0", "s0", "t0", "m0", "x0", "k0"])
    path = write_v3(seg, str(tmp_path))
    back = load_v3(path)
    assert back.num_docs == seg.num_docs and list(back.columns) == list(seg.columns)
    for n, c in seg.columns.items():
        b = back.columns[n]
        assert (b.data_type, b.has_dictionary, b.is_sorted, b.cardinality, b.bits_per_element, b.dict_entry_bytes) == \
            (c.data_type, c.has_dictionary, c.is_sorted, c.cardinality, c.bits_per_element, c.dict_entry_bytes)
        assert (b.forward_index == c.forward_index).all()
        assert (b.inverted_index is None) == (c.inverted_index is None)
    assert any(b.forward_index.ctypes.data % 4 for b in back.columns.values())      # really unaligned views
    d3 = seg.columns["c3"].dictionary_values()
    for sql in (f"SELECT s0, COUNT(*), SUM(m0), MAX(x0) FROM t WHERE c3 IN ({int(d3[2])}, {int(d3[9])}) OR t0 = 20005 GROUP BY s0 LIMIT 100000",
                "SELECT d0, DISTINCTCOUNT(c1), MIN(k0) FROM t WHERE x0 < 0.5 GROUP BY d0"):
        q = parse_sql(sql)
        a, b = oracle.execute(seg, q), oracle.execute(back, q)
        assert a.stats == b.stats and a.decoded_keys() == b.decoded_keys()
        assert all((x == y).all() for x, y in zip(a.doubles, b.doubles)) and all((x == y).all() for x, y in zip(a.longs, b.longs))


def test_var_length_string_dictionary_roundtrip_and_oracle():
    """.vl; dictionaries (VarLengthValueWriter.java:78-125 / VarLengthValueReader.java:41-96): same values, same dictIds,
    same query results as the fixed-width form of the same column -- in the writer's reader, the oracle, and the lowering
    of the host planning layer (which sees the stager's padded copy)."""
    from oracle import oracle
    from pinot_b200 import native
    from pinot_b200.query import parse_sql
    from pinot_b200.segment_writer import DataType, build_column, is_var_length_dictionary, make_segment
    rng = np.random.Generator(np.random.PCG64(7))
    words = [b"a", b"ab", b"abc", b"zebra", b"pinot-b200", b"x" * 37, b"mid", b"", b"q"]
    vals = [words[i] for i in rng.integers(0, len(words), size=5000)]
    nums = rng.integers(0, 1000, size=5000)
    segs = {}
    for vl in (False, True):
        cols = [build_column("s", DataType.STRING, vals, var_length_dictionary=vl, inverted=True),
                build_column("v", DataType.INT, nums)]
        segs[vl] = make_segment("vl" if vl else "fixed", cols)
    assert is_var_length_dictionary(segs[True].columns["s"].dictionary) and not is_var_length_dictionary(segs[False].columns["s"].dictionary)
    assert list(segs[True].columns["s"].dictionary_values()) == list(segs[False].columns["s"].dictionary_values()) == sorted(set(words))
    staged = {vl: native.SegmentGroup([native.StagedSegment(segs[vl])]) for vl in (False, True)}
    for sql in ("SELECT s, COUNT(*), SUM(v) FROM t WHERE s > 'ab' AND s <= 'pinot-b200' GROUP BY s LIMIT 100",
                "SELECT COUNT(*), MAX(v) FROM t WHERE s IN ('', 'zebra', 'nosuch') OR s = 'mid'",
                "SELECT s, DISTINCTCOUNT(v) FROM t WHERE s != 'q' GROUP BY s LIMIT 100"):
        q = parse_sql(sql)
        a, b = oracle.execute(segs[False], q), oracle.execute(segs[True], q)
        assert a.decoded_keys() == b.decoded_keys() and a.stats == b.stats
        for x, y in zip(a.doubles + a.longs, b.doubles + b.longs):
            assert np.array_equal(x, y)
        assert native.dump_lowered(staged[False], q) == native.dump_lowered(staged[True], q)


# ---- chunk codecs of raw forward indexes (ChunkCompressionType LZ4 / LZ4_LENGTH_PREFIXED / SNAPPY) ----

def test_lz4_block_known_answers():
    """Hand-assembled streams of the public LZ4 block format (what lz4-java's safeDecompressor reads, LZ4Decompressor.java:41-52)."""
    dec = lambda b, n: oracle.block_decode("lz4", bytes(b), n)
    assert dec([0x50] + list(b"hello"), 5) == b"hello"                                  # literals only: token 5:0
    # 'a', then a match at offset 1 of length 4 + 5 that overlaps its own output (run-length), then 5 closing literals
    assert dec([0x15, ord("a"), 0x01, 0x00, 0x50] + list(b"bcdef"), 15) == b"a" * 10 + b"bcdef"
    # 'abcd', match offset 4 length 4 + 15 + 7 (length extension byte), closing literal
    assert dec([0x4F] + list(b"abcd") + [0x04, 0x00, 0x07, 0x10, ord("z")], 31) == b"abcd" * 7 + b"ab" + b"z"
    # 15 + 255 + 3 literals through two length-extension bytes
    lit = bytes(range(256)) + bytes(17)
    assert dec([0xF0, 0xFF, 0x03] + list(lit), len(lit)) == lit
    for bad in ([0x15, ord("a"), 0x00, 0x00, 0x10, 0], [0x15, ord("a"), 0x05, 0x00, 0x10, 0], [0x60, 1, 2]):   # offset 0, offset before the start, truncated
        with pytest.raises(ValueError):
            dec(bad, 64)


def test_snappy_block_known_answers():
    dec = lambda b, n: oracle.block_decode("snappy", bytes(b), n)
    assert dec([5, (5 - 1) << 2] + list(b"hello"), 5) == b"hello"
    # literal 'ab', then copy-1 (tag 01) of length 4 + 3 = 7 at offset 2: 'ababababa'
    assert dec([9, (2 - 1) << 2] + list(b"ab") + [(3 << 2) | 1, 2], 9) == b"ababababa"
    # literal 'xyz', copy-2 (tag 10) length 6 at offset 3
    assert dec([9, (3 - 1) << 2] + list(b"xyz") + [((6 - 1) << 2) | 2, 3, 0], 9) == b"xyzxyzxyz"
    # literal of 100 bytes: length - 1 = 99 in one extra byte (tag 60 << 2)
    lit = bytes(range(100))
    assert dec([100, 60 << 2, 99] + list(lit), 100) == lit
    with pytest.raises(ValueError):
        dec([9, (2 - 1) << 2] + list(b"ab") + [(3 << 2) | 1, 3], 9)                      # offset before the start


@pytest.mark.parametrize("codec", ["lz4", "snappy"])
def test_block_decoders_against_the_stock_libraries(codec):
    """The oracle's decoders against liblz4 / libsnappy (through pyarrow): random, repetitive and mixed payloads."""
    pa = pytest.importorskip("pyarrow")
    name = {"lz4": "lz4_raw", "snappy": "snappy"}[codec]
    rng = np.random.default_rng(5)
    payloads = [b"", b"x", bytes(11), rng.integers(0, 256, 70000, dtype=np.uint8).tobytes(), (b"pinot" * 30000)[:99991],
                np.repeat(rng.integers(0, 50, 3000), rng.integers(1, 40, 3000)).astype(">i4").tobytes(),
                np.cumsum(rng.integers(0, 3, 20000)).astype(">i8").tobytes(), bytes(200000)]
    for p in payloads:
        z = pa.Codec(name).compress(p, asbytes=True)
        assert oracle.block_decode(codec, z, len(p)) == p


@pytest.mark.parametrize("compression", ["LZ4", "LZ4_LENGTH_PREFIXED", "SNAPPY"])
@pytest.mark.parametrize("version", [2, 3, 4])
def test_compressed_raw_forward_index(compression, version):
    """BaseChunkForwardIndexWriter framing (header, per-chunk offsets, independently compressed chunks, short last chunk) and
    the oracle's rewrite to PASS_THROUGH: same values as the uncompressed index of the same column."""
    rng = np.random.default_rng(version)
    n = 2 * 1000 + 137
    for dt, vals in ((DataType.LONG, np.cumsum(rng.integers(-3, 50, n)).astype(np.int64)), (DataType.INT, rng.integers(-9, 9, n).astype(np.int32)),
                     (DataType.DOUBLE, np.round(rng.normal(0, 10, n), 1)), (DataType.FLOAT, rng.integers(0, 4, n).astype(np.float32))):
        plain = build_column("k", dt, vals, dictionary=False, raw_version=version)
        comp = build_column("k", dt, vals, dictionary=False, raw_compression=compression, raw_version=version)
        raw = comp.forward_index.tobytes()
        v, num_chunks, per_chunk, width, total, codec, header_start = struct.unpack_from(">7i", raw, 0)
        assert (v, num_chunks, per_chunk, total, header_start) == (version, 3, 1000, n, 28)
        assert codec == {"LZ4": 3, "LZ4_LENGTH_PREFIXED": 4, "SNAPPY": 1}[compression]
        offs = struct.unpack_from(">3i" if version == 2 else ">3q", raw, 28)
        assert offs[0] == 28 + 3 * (4 if version == 2 else 8) and offs[0] < offs[1] < offs[2] < len(raw)
        assert comp.forward_index.size < plain.forward_index.size or dt == DataType.DOUBLE
        out = oracle.raw_forward_decompress(comp.forward_index, width)
        assert out.tobytes() == plain.forward_index.tobytes()


def test_oracle_reads_compressed_raw_columns():
    from pinot_b200.query import parse_sql
    from pinot_b200.segment_writer import make_segment
    rng = np.random.default_rng(9)
    n = 5000
    d = rng.integers(0, 7, n).astype(np.int32)
    k = rng.integers(-1000, 1000, n).astype(np.int64)
    x = np.round(rng.normal(0, 5, n), 2)
    def seg(compression):
        return make_segment("s", [build_column("d", DataType.INT, d), build_column("k", DataType.LONG, k, dictionary=False, raw_compression=compression),
                                  build_column("x", DataType.DOUBLE, x, dictionary=False, raw_compression=compression)])
    q = parse_sql("SELECT d, COUNT(*), SUM(k), MAX(x), DISTINCTCOUNT(k) FROM t WHERE k > -500 AND x < 4.5 GROUP BY d LIMIT 100")
    ref = oracle.execute(seg(None), q)
    for compression in ("LZ4", "LZ4_LENGTH_PREFIXED", "SNAPPY"):
        got = oracle.execute(seg(compression), q)
        assert got.stats == ref.stats and got.decoded_keys() == ref.decoded_keys()
        for a in range(len(q.aggregations)):
            assert np.array_equal(got.doubles[a], ref.doubles[a]) and np.array_equal(got.longs[a], ref.longs[a])


# ---- null-value vectors (IS NULL / IS NOT NULL: FilterPlanNode.java:294-307, BitmapBasedFilterOperator) ----

def _null_segment(n=20_000, seed=4):
    from pinot_b200.segment_writer import make_segment, with_nulls
    rng = np.random.default_rng(seed)
    i_null = rng.random(n) < 0.13
    k_null = np.zeros(n, dtype=bool); k_null[5000:5400] = True; k_null[::97] = True        # a run container and scattered docs
    i = np.where(i_null, np.iinfo(np.int32).min, rng.integers(0, 50, n)).astype(np.int32)   # default null value of an INT dimension
    k = np.where(k_null, 0, rng.integers(1, 1_000_000, n)).astype(np.int64)
    d = rng.integers(0, 6, n).astype(np.int32)
    seg = make_segment("nulls", [build_column("d", DataType.INT, d), with_nulls(build_column("i", DataType.INT, i), i_null),
                                 with_nulls(build_column("k", DataType.LONG, k, dictionary=False), k_null),
                                 with_nulls(build_column("z", DataType.INT, d), np.zeros(n, dtype=bool))])
    return seg, d, i, k, i_null, k_null


def test_null_value_vector_layout_and_v3(tmp_path):
    from pinot_b200.segment_writer import load_v3, write_v3
    seg, d, i, k, i_null, k_null = _null_segment()
    assert seg.columns["z"].null_value_vector is None                       # NullValueVectorCreator.seal: no file for an empty bitmap
    got = np.zeros(seg.num_docs * 2, dtype=np.uint32)
    v = seg.columns["k"].null_value_vector
    n = oracle.lib().orc_roaring_to_doc_ids(v.ctypes.data, v.size, got.ctypes.data, got.size)
    assert np.array_equal(got[:n], np.flatnonzero(k_null))
    back = load_v3(write_v3(seg, str(tmp_path)))
    assert back.columns["i"].null_value_vector.tobytes() == seg.columns["i"].null_value_vector.tobytes()
    assert back.columns["d"].null_value_vector is None


def test_oracle_is_null_predicates():
    """SegmentWithNullValueVectorTest.testNotNullPredicate / testNullPredicate / testNullWithAndPredicate (:242-273): counts
    against the generated data; plus OR / NOT around the bitmap leaves and a column without a vector."""
    from pinot_b200.query import parse_sql
    seg, d, i, k, i_null, k_null = _null_segment()
    n = seg.num_docs
    cnt = lambda sql: int(oracle.execute(seg, parse_sql(sql)).longs[0][0])
    assert cnt("SELECT COUNT(*) FROM t WHERE i IS NOT NULL") == n - int(i_null.sum())
    assert cnt("SELECT COUNT(*) FROM t WHERE i IS NULL") == int(i_null.sum())
    assert cnt("SELECT COUNT(*) FROM t WHERE i IS NOT NULL AND k > 500000") == int((~i_null & (k > 500000)).sum())
    assert cnt("SELECT COUNT(*) FROM t WHERE i IS NULL OR k IS NULL") == int((i_null | k_null).sum())
    assert cnt("SELECT COUNT(*) FROM t WHERE NOT (i IS NULL) AND k IS NULL AND d < 3") == int((~i_null & k_null & (d < 3)).sum())
    assert cnt("SELECT COUNT(*) FROM t WHERE z IS NULL") == 0 and cnt("SELECT COUNT(*) FROM t WHERE z IS NOT NULL") == n
    r = oracle.execute(seg, parse_sql("SELECT d, COUNT(*), SUM(k) FROM t WHERE k IS NOT NULL AND i IS NULL GROUP BY d LIMIT 10"))
    m = ~k_null & i_null
    exp = {int(g): (int((m & (d == g)).sum()), float(k[m & (d == g)].sum())) for g in np.unique(d[m])}
    assert {key[0]: (int(c), float(s)) for key, c, s in zip(r.decoded_keys(), r.longs[0], r.doubles[1])} == exp
    assert r.stats["num_entries_scanned_in_filter"] == 0                     # bitmap-based leaves scan nothing
