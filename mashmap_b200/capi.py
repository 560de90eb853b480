"""ctypes binding of the C ABI in include/mashmap_b200.h (tests, bench.py, smoke()).

The product is the C++/CUDA code behind the ABI; this module only marshals numpy arrays into it.
Import fails loudly when the in-tree CUDA library has not been built -- there is no Python or
CPU implementation to fall back to.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmashmap_b200.so")

MM_OK, MM_EINVAL, MM_ENODEVICE, MM_ECUDA, MM_ENOMEM, MM_ECAPACITY, MM_ESTATE = 0, -1, -2, -3, -4, -5, -6
MM_KEEP_LOOKUP, MM_KEEP_UNFILTERED = 1, 2

# record layouts == include/mashmap_b200.h
minmer_dtype = np.dtype(
    [("hash", "<u8"), ("wpos", "<i4"), ("wpos_end", "<i4"), ("seqId", "<i4"), ("strand", "<i2"), ("_pad", "<i2")]
)
ipoint_dtype = np.dtype(
    [("pos", "<i4"), ("_pad0", "<i4"), ("hash", "<u8"), ("seqId", "<i4"), ("side", "i1"), ("_pad1", "i1", (3,))]
)
l1_dtype = np.dtype(
    [("seqId", "<i4"), ("rangeStartPos", "<i4"), ("rangeEndPos", "<i4"), ("intersectionSize", "<i4"),
     ("segment", "<u4"), ("first_locus", "<u4"), ("n_loci", "<u4"), ("_pad", "<u4")]
)
l2_dtype = np.dtype(
    [("seqId", "<i4"), ("meanOptimalPos", "<i4"), ("optimalStart", "<i4"), ("optimalEnd", "<i4"),
     ("sharedSketchSize", "<i4"), ("strand", "<i4")]
)
segres_dtype = np.dtype(
    [("sketch_max_hash", "<u8"), ("sketch_raw_count", "<i4"), ("sketch_size", "<i4"), ("n_points", "<i4"),
     ("minimum_hits", "<i4"), ("best_intersection", "<i4"), ("first_candidate", "<u4"), ("n_candidates", "<u4"),
     ("_pad", "<u4")]
)
segment_dtype = np.dtype(
    [("offset", "<u8"), ("length", "<i4"), ("seq_counter", "<i4"), ("name_id", "<i4"), ("ref_group", "<i4")]
)
assert minmer_dtype.itemsize == 24 and ipoint_dtype.itemsize == 24 and l1_dtype.itemsize == 32
assert l2_dtype.itemsize == 24 and segres_dtype.itemsize == 40 and segment_dtype.itemsize == 24


class Params(C.Structure):
    _fields_ = [
        ("kmer_size", C.c_int32), ("seg_length", C.c_int32), ("sketch_size", C.c_int32),
        ("stage1_topani_filter", C.c_int32), ("skip_self", C.c_int32), ("skip_prefix", C.c_int32),
        ("lower_triangular", C.c_int32), ("_reserved", C.c_int32 * 9),
    ]


class MashmapError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"mashmap_b200 error {code}: {msg}")
        self.code = code


class IndexStats(C.Structure):
    """mm_index_stats"""
    _fields_ = [("n_minmers", C.c_uint64), ("n_minmers_before_filter", C.c_uint64), ("n_keys", C.c_uint64), ("n_points", C.c_uint64),
                ("freq_threshold", C.c_int32), ("n_chunks", C.c_uint32), ("n_fixed_chunks", C.c_uint32), ("fix_rounds", C.c_uint32),
                ("hist_min_count", C.c_uint32), ("hist_max_count", C.c_uint32), ("hist_min_keys", C.c_uint64), ("hist_max_keys", C.c_uint64),
                ("ms_scan", C.c_float), ("ms_post", C.c_float), ("ms_lookup", C.c_float), ("ms_total", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class FastqRecords(C.Structure):
    _fields_ = [("n_records", C.c_uint64), ("name_off", C.POINTER(C.c_uint64)), ("seq_len", C.POINTER(C.c_uint64)),
                ("nib_off", C.POINTER(C.c_uint64)), ("names", C.c_void_p), ("nibbles", C.c_void_p), ("consumed", C.c_uint64),
                ("ended", C.c_int)]


_lib = None


def lib():
    """Load the CUDA library; raise (never fall back) if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(mashmap_b200 has no CPU implementation)"
            )
        L = C.CDLL(LIB_PATH)
        vp, u64, i32 = C.c_void_p, C.c_uint64, C.c_int32
        L.mm_ctx_create.argtypes = [C.c_int, C.POINTER(Params), C.POINTER(vp)]
        L.mm_ctx_destroy.argtypes = [vp]
        L.mm_ctx_device.argtypes = [vp]
        L.mm_last_error.argtypes = [vp]
        L.mm_last_error.restype = C.c_char_p
        L.mm_kernel_launches.argtypes = [vp]
        L.mm_kernel_launches.restype = u64
        L.mm_ctx_diag.argtypes = [vp, C.POINTER(u64 * 8)]
        L.mm_index_upload.argtypes = [vp, vp, u64, vp, vp, u64, vp, u64, vp, vp, vp, vp, i32]
        L.mm_tables_upload.argtypes = [vp, vp, i32, vp, i32]
        L.mm_index_build.argtypes = [vp, vp, C.c_int, vp, i32, vp, vp, C.c_float, C.c_int, C.POINTER(IndexStats)]
        L.mm_index_download.argtypes = [vp, vp, vp, vp, vp, vp]
        L.mm_index_build_minmers.argtypes = [vp, vp, u64, C.c_int, vp, vp, vp, i32, C.c_float, C.c_int, C.POINTER(IndexStats)]
        L.mm_index_download_unfiltered.argtypes = [vp, vp, u64, C.POINTER(u64)]
        L.mm_index_release_kept.argtypes = [vp]
        L.mm_index_blob.argtypes = [vp, C.POINTER(vp), C.POINTER(u64)]
        L.mm_index_blob_alloc.argtypes = [vp, u64, C.POINTER(vp)]
        L.mm_index_adopt_blob.argtypes = [vp]
        L.mm_ctx_share_index.argtypes = [vp, vp]
        L.mm_sketch_segments.argtypes = [vp, vp, u64, vp, u64, vp, vp]
        L.mm_map_segments.argtypes = [vp, vp, u64, vp, u64, vp, vp, u64, C.POINTER(u64), vp, u64, C.POINTER(u64)]
        L.mm_batch_upload.argtypes = [vp, vp, u64, vp, u64]
        L.mm_batch_upload_packed.argtypes = [vp, vp, u64, vp, u64]
        L.mm_map_segments_packed.argtypes = [vp, vp, u64, vp, u64, vp, vp, u64, C.POINTER(u64), vp, u64, C.POINTER(u64)]
        L.mm_last_pack_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L.mm_map_resident.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
        L.mm_map_resident_l1_best.argtypes = [vp, vp]
        L.mm_map_resident_with_best.argtypes = [vp, vp, vp, C.POINTER(u64), C.POINTER(u64)]
        L.mm_index_key_counts.argtypes = [vp, vp, C.c_int, vp, i32, vp, vp, u64, C.POINTER(u64), C.POINTER(IndexStats)]
        L.mm_index_build_shard.argtypes = [vp, vp, C.c_int, vp, i32, i32, vp, vp, vp, i32, vp, u64, C.c_int, C.POINTER(IndexStats)]
        L.mm_batch_fetch.argtypes = [vp, vp, vp, u64, vp, u64]
        L.mm_batch_fetch_sketch.argtypes = [vp, vp, vp]
        L.mm_last_stage_ms.argtypes = [vp, C.POINTER(C.c_float * 8)]
        L.mm_host_alloc.argtypes = [C.POINTER(vp), u64]
        L.mm_host_free.argtypes = [vp]
        L.mm_inflater_create.argtypes = [C.c_int, C.POINTER(vp)]
        L.mm_inflater_destroy.argtypes = [vp]
        L.mm_inflater_error.argtypes = [vp]
        L.mm_inflater_error.restype = C.c_char_p
        L.mm_inflate_blocks.argtypes = [vp, vp, vp, vp, vp, u64, vp, C.POINTER(C.c_int64)]
        L.mm_inflater_last_ms.argtypes = [vp, C.POINTER(C.c_float * 2)]
        L.mm_fastq_create.argtypes = [C.c_int, C.POINTER(vp)]
        L.mm_fastq_destroy.argtypes = [vp]
        L.mm_fastq_error.argtypes = [vp]
        L.mm_fastq_error.restype = C.c_char_p
        L.mm_fastq_append_text.argtypes = [vp, vp, u64]
        L.mm_fastq_append_blocks.argtypes = [vp, vp, vp, vp, vp, u64, C.POINTER(C.c_int64)]
        L.mm_fastq_cut.argtypes = [vp, C.c_int, C.POINTER(FastqRecords)]
        L.mm_fastq_last_ms.argtypes = [vp, C.POINTER(C.c_float * 2)]
        _lib = L
    return _lib


EXPORTED_SYMBOLS = [
    "mm_ctx_create", "mm_ctx_destroy", "mm_ctx_device", "mm_last_error", "mm_kernel_launches", "mm_ctx_diag", "mm_index_upload",
    "mm_tables_upload", "mm_index_build", "mm_index_download", "mm_index_blob", "mm_index_blob_alloc", "mm_index_adopt_blob", "mm_ctx_share_index", "mm_sketch_segments",
    "mm_map_segments", "mm_map_segments_packed", "mm_batch_upload", "mm_batch_upload_packed", "mm_last_pack_ms", "mm_map_resident", "mm_batch_fetch", "mm_batch_fetch_sketch",
    "mm_last_stage_ms", "mm_ctx_set_phase_hook", "mm_ctx_set_wait_mode", "mm_params_check", "mm_host_alloc", "mm_host_free",
    "mm_index_key_counts", "mm_index_build_shard", "mm_map_resident_l1_best", "mm_map_resident_with_best",
    "mm_inflater_create", "mm_inflater_destroy", "mm_inflater_error", "mm_inflate_blocks", "mm_inflater_last_ms",
    "mm_fastq_create", "mm_fastq_destroy", "mm_fastq_error", "mm_fastq_append_text", "mm_fastq_append_blocks", "mm_fastq_cut",
    "mm_fastq_last_ms", "mm_index_build_minmers", "mm_index_download_unfiltered", "mm_index_release_kept",
]


def params_check(kmer_size, seg_length, sketch_size):
    """mm_params_check: (MM_OK, "") if a context with these parameters can launch every mapping kernel, else (MM_EINVAL,
    the message naming the kernel that does not fit). Needs no device."""
    L = lib()
    rc = L.mm_params_check(C.byref(Params(kmer_size, seg_length, sketch_size)))
    return rc, ("" if rc == MM_OK else L.mm_last_error(None).decode())


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _keep(keep_lookup, keep_unfiltered):
    return (MM_KEEP_LOOKUP if keep_lookup else 0) | (MM_KEEP_UNFILTERED if keep_unfiltered else 0)


def _c(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    return a


_NIB = np.full(256, 8, dtype=np.uint8)
for _ch, _code in ((b"A", 0), (b"C", 1), (b"T", 2), (b"G", 3)):
    _NIB[_ch[0]] = _code
    _NIB[_ch.lower()[0]] = _code


def pack_bases(ascii_bases):
    """numpy statement of the device input format (include/mashmap_b200.h, mm_map_segments_packed): one nibble per base,
    2-bit code (A 0, C 1, T 2, G 3) | 8 for anything that is not ACGT after upper-casing; base i in byte i // 2, low
    nibble first. Used by the tests; the product packs in C++ (skch::BatchMapper) or on the device (k_pack_bases)."""
    a = np.ascontiguousarray(ascii_bases, dtype=np.uint8)
    n = _NIB[a]
    if len(n) & 1:
        n = np.concatenate([n, np.array([8], dtype=np.uint8)])
    return (n[0::2] | (n[1::2] << 4)).astype(np.uint8)


class PinnedBuffer:
    """Page-locked host memory exposed as a numpy uint8 array."""

    def __init__(self, nbytes):
        self.ptr = C.c_void_p()
        rc = lib().mm_host_alloc(C.byref(self.ptr), max(int(nbytes), 1))
        if rc != MM_OK:
            raise MashmapError(rc, "mm_host_alloc failed")
        self.nbytes = int(nbytes)
        self.array = np.ctypeslib.as_array(C.cast(self.ptr, C.POINTER(C.c_uint8)), shape=(max(self.nbytes, 1),))

    def free(self):
        if self.ptr:
            lib().mm_host_free(self.ptr)
            self.ptr = C.c_void_p()

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Inflater:
    """mm_inflater: raw DEFLATE blocks inflated on the device"""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = lib().mm_inflater_create(device, C.byref(self._h))
        if rc != MM_OK:
            raise MashmapError(rc, lib().mm_inflater_error(None).decode())

    def inflate(self, comp, comp_off, out_off, crc, out=None):
        """(rc, bad_block, out, error): comp uint8, comp_off / out_off uint64 [n+1], crc uint32 [n]"""
        comp = _c(comp, np.uint8)
        comp_off, out_off, crc = _c(comp_off, np.uint64), _c(out_off, np.uint64), _c(crc, np.uint32)
        n = len(crc)
        if out is None:
            out = np.zeros(max(int(out_off[-1]) if n else 0, 1), dtype=np.uint8)
        bad = C.c_int64()
        rc = lib().mm_inflate_blocks(self._h, _ptr(comp), _ptr(comp_off), _ptr(out_off), _ptr(crc), n, _ptr(out), C.byref(bad))
        return rc, bad.value, out, lib().mm_inflater_error(self._h).decode()

    def last_ms(self):
        a = (C.c_float * 2)()
        lib().mm_inflater_last_ms(self._h, C.byref(a))
        return a[0], a[1]

    def close(self):
        if self._h:
            lib().mm_inflater_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class FastqParser:
    """mm_fastq: a window of FASTQ text in device memory, cut into records and packed to nibbles on the device"""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = lib().mm_fastq_create(device, C.byref(self._h))
        if rc != MM_OK:
            raise MashmapError(rc, lib().mm_fastq_error(None).decode())

    def _check(self, rc, what):
        if rc != MM_OK:
            raise MashmapError(rc, f"{what}: " + lib().mm_fastq_error(self._h).decode())

    def append_text(self, text):
        a = np.frombuffer(bytes(text), dtype=np.uint8)
        self._check(lib().mm_fastq_append_text(self._h, _ptr(a), len(a)), "mm_fastq_append_text")

    def append_blocks(self, comp, comp_off, out_off, crc):
        """(rc, bad_block, error): BGZF member data inflated straight into the window"""
        comp = _c(comp, np.uint8)
        comp_off, out_off, crc = _c(comp_off, np.uint64), _c(out_off, np.uint64), _c(crc, np.uint32)
        bad = C.c_int64()
        rc = lib().mm_fastq_append_blocks(self._h, _ptr(comp), _ptr(comp_off), _ptr(out_off), _ptr(crc), len(crc), C.byref(bad))
        return rc, bad.value, lib().mm_fastq_error(self._h).decode()

    def cut(self, last):
        """dict of the cut's records, copied out of the handle's buffers: names [bytes], seq_len, nibbles [bytes per
        record], consumed, ended"""
        r = FastqRecords()
        self._check(lib().mm_fastq_cut(self._h, int(last), C.byref(r)), "mm_fastq_cut")
        n = int(r.n_records)
        noff = np.ctypeslib.as_array(r.name_off, shape=(n + 1,)).copy() if n else np.zeros(1, np.uint64)
        boff = np.ctypeslib.as_array(r.nib_off, shape=(n + 1,)).copy() if n else np.zeros(1, np.uint64)
        slen = np.ctypeslib.as_array(r.seq_len, shape=(n,)).copy() if n else np.zeros(0, np.uint64)
        names = C.string_at(r.names, int(noff[-1])) if n else b""
        nib = C.string_at(r.nibbles, int(boff[-1])) if n else b""
        return {"names": [names[int(noff[i]):int(noff[i + 1])] for i in range(n)], "seq_len": slen,
                "nibbles": [nib[int(boff[i]):int(boff[i + 1])] for i in range(n)], "nib_off": boff, "nib_all": nib,
                "consumed": int(r.consumed), "ended": int(r.ended)}

    def last_ms(self):
        a = (C.c_float * 2)()
        lib().mm_fastq_last_ms(self._h, C.byref(a))
        return a[0], a[1]

    def close(self):
        if self._h:
            lib().mm_fastq_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Context:
    def __init__(self, device=0, kmer_size=19, seg_length=5000, sketch_size=220, stage1_topani_filter=True,
                 skip_self=False, skip_prefix=False, lower_triangular=False):
        self._L = lib()
        self.params = Params(kmer_size, seg_length, sketch_size, int(stage1_topani_filter), int(skip_self),
                             int(skip_prefix), int(lower_triangular))
        self._h = C.c_void_p()
        rc = self._L.mm_ctx_create(device, C.byref(self.params), C.byref(self._h))
        if rc != MM_OK:
            raise MashmapError(rc, self._L.mm_last_error(None).decode())
        self.sketch_size = sketch_size
        self.device = device

    @classmethod
    def from_handle(cls, handle, sketch_size, device=0):
        """wrap an mm_ctx owned by someone else (the host library's BatchMapper); close() will not destroy it"""
        self = cls.__new__(cls)
        self._L = lib()
        self._h = C.c_void_p(handle)
        self._borrowed = True
        self.sketch_size = sketch_size
        self.device = device
        return self

    def close(self):
        if self._h and not getattr(self, "_borrowed", False):
            self._L.mm_ctx_destroy(self._h)
        self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != MM_OK:
            raise MashmapError(rc, self._L.mm_last_error(self._h).decode())

    DIAG_NAMES = ("l1_cta_segments", "l1_pool_regrow", "cand_regrow", "l2_general_cands", "l2_loci_regrow", "sketch_general_segments",
                  "long_fragments")

    def diag(self):
        """how often the rare paths ran (mm_ctx_diag), by name"""
        out = (C.c_uint64 * 8)()
        self._check(self._L.mm_ctx_diag(self._h, C.byref(out)))
        return {n: int(out[i]) for i, n in enumerate(self.DIAG_NAMES)}

    @property
    def kernel_launches(self):
        return int(self._L.mm_kernel_launches(self._h))

    def index_upload(self, minmers, keys, offsets, points, key_is_freq, contig_len, contig_name_id=None,
                     contig_group=None):
        minmers = _c(minmers, minmer_dtype)
        keys = _c(keys, np.uint64)
        offsets = _c(offsets, np.uint64)
        points = _c(points, ipoint_dtype)
        key_is_freq = _c(key_is_freq, np.uint8)
        contig_len = _c(contig_len, np.int32)
        cn = None if contig_name_id is None else _c(contig_name_id, np.int32)
        cg = None if contig_group is None else _c(contig_group, np.int32)
        self._check(self._L.mm_index_upload(self._h, _ptr(minmers), len(minmers), _ptr(keys), _ptr(offsets), len(keys),
                                            _ptr(points), len(points), _ptr(key_is_freq), _ptr(contig_len), _ptr(cn),
                                            _ptr(cg), len(contig_len)))

    def index_build(self, seqs, contig_offsets, contig_name_id=None, contig_group=None, kmer_pct_threshold=0.001, keep_lookup=False,
                    device_ptr=None, keep_unfiltered=False):
        """mm_index_build: the reference index built on the device. seqs: uint8 array (contigs back to back) on the host, or
        pass device_ptr (int) for text that is already in device memory. Returns the statistics as a dict."""
        offs = _c(contig_offsets, np.uint64)
        n = len(offs) - 1
        cn = None if contig_name_id is None else _c(contig_name_id, np.int32)
        cg = None if contig_group is None else _c(contig_group, np.int32)
        keep = _keep(keep_lookup, keep_unfiltered)
        st = IndexStats()
        if device_ptr is not None:
            rc = self._L.mm_index_build(self._h, C.c_void_p(int(device_ptr)), 1, _ptr(offs), n, _ptr(cn), _ptr(cg), kmer_pct_threshold,
                                        keep, C.byref(st))
        else:
            a = np.ascontiguousarray(seqs, dtype=np.uint8)
            rc = self._L.mm_index_build(self._h, _ptr(a), 0, _ptr(offs), n, _ptr(cn), _ptr(cg), kmer_pct_threshold,
                                        keep, C.byref(st))
        self._check(rc)
        self._index_stats = st.as_dict()
        return self._index_stats

    def index_build_minmers(self, minmers, contig_len, contig_name_id=None, contig_group=None, kmer_pct_threshold=0.001,
                            keep_lookup=False, keep_unfiltered=False, device_ptr=None):
        """mm_index_build_minmers: the index built on the device from a minmer list as --saveIndex writes it (minmer_dtype,
        host), or from device_ptr (int) holding len(minmers) such records in device memory. Returns the statistics."""
        n = len(minmers)
        cl = _c(contig_len, np.int32)
        cn = None if contig_name_id is None else _c(contig_name_id, np.int32)
        cg = None if contig_group is None else _c(contig_group, np.int32)
        st = IndexStats()
        if device_ptr is not None:
            src, on_device = C.c_void_p(int(device_ptr)), 1
        else:
            mi = _c(minmers, minmer_dtype)
            src, on_device = _ptr(mi), 0
        self._check(self._L.mm_index_build_minmers(self._h, src, n, on_device, _ptr(cl), _ptr(cn), _ptr(cg), len(cl), kmer_pct_threshold,
                                                   _keep(keep_lookup, keep_unfiltered), C.byref(st)))
        self._index_stats = st.as_dict()
        return self._index_stats

    def index_download_unfiltered(self):
        """mm_index_download_unfiltered: the records a build kept with keep_unfiltered=True (before the frequent-seed drop)"""
        n = C.c_uint64()
        rc = self._L.mm_index_download_unfiltered(self._h, None, 0, C.byref(n))
        out = np.zeros(n.value, dtype=minmer_dtype)
        if rc == MM_ECAPACITY:
            rc = self._L.mm_index_download_unfiltered(self._h, _ptr(out), n.value, C.byref(n))
        self._check(rc)
        return out

    def index_release_kept(self):
        """mm_index_release_kept: free what keep_lookup / keep_unfiltered kept on the device"""
        self._check(self._L.mm_index_release_kept(self._h))

    def index_key_counts(self, seqs, contig_offsets):
        """pass 1 of a contig-sharded index (mm_index_key_counts): (distinct hashes ascending, their interval-point counts,
        statistics) of the contigs seqs / contig_offsets"""
        a = np.ascontiguousarray(seqs, dtype=np.uint8)
        offs = _c(contig_offsets, np.uint64)
        n, st = C.c_uint64(), IndexStats()
        rc = self._L.mm_index_key_counts(self._h, _ptr(a), 0, _ptr(offs), len(offs) - 1, None, None, 0, C.byref(n), C.byref(st))
        keys, counts = np.zeros(n.value, dtype=np.uint64), np.zeros(n.value, dtype=np.uint32)
        if rc == MM_ECAPACITY:
            rc = self._L.mm_index_key_counts(self._h, None, 0, None, 0, _ptr(keys), _ptr(counts), n.value, C.byref(n), None)
        self._check(rc)
        return keys, counts, st.as_dict()

    def index_build_shard(self, seqs, contig_offsets, first_contig, contig_len, freq_hashes, contig_name_id=None,
                          contig_group=None, keep_lookup=False):
        """pass 2 (mm_index_build_shard): the image of contigs [first_contig, first_contig + len(contig_offsets) - 1) of a
        reference whose contig lengths are contig_len (all of them), with exactly freq_hashes (ascending) frequent"""
        a = np.ascontiguousarray(seqs, dtype=np.uint8)
        offs = _c(contig_offsets, np.uint64)
        cl = _c(contig_len, np.int32)
        fr = _c(freq_hashes, np.uint64)
        cn = None if contig_name_id is None else _c(contig_name_id, np.int32)
        cg = None if contig_group is None else _c(contig_group, np.int32)
        st = IndexStats()
        self._check(self._L.mm_index_build_shard(self._h, _ptr(a), 0, _ptr(offs), int(first_contig), len(offs) - 1, _ptr(cl),
                                                 _ptr(cn), _ptr(cg), len(cl), _ptr(fr), len(fr), 1 if keep_lookup else 0,
                                                 C.byref(st)))
        self._index_stats = st.as_dict()
        return self._index_stats

    def index_download(self):
        """host copies of the device-built index (needs keep_lookup=True): (minmers, keys, offsets, points, is_freq)"""
        st = self._index_stats
        mi = np.zeros(st["n_minmers"], dtype=minmer_dtype)
        keys = np.zeros(st["n_keys"], dtype=np.uint64)
        offs = np.zeros(st["n_keys"] + 1, dtype=np.uint64)
        pts = np.zeros(st["n_points"], dtype=ipoint_dtype)
        fr = np.zeros(st["n_keys"], dtype=np.uint8)
        self._check(self._L.mm_index_download(self._h, _ptr(mi), _ptr(keys), _ptr(offs), _ptr(pts), _ptr(fr)))
        return mi, keys, offs, pts, fr

    def index_minmers(self):
        """host copy of the device index's minmerIndex records only (needs no keep_lookup)"""
        n = int(self._index_stats["n_minmers"]) if getattr(self, "_index_stats", None) else 0
        if n == 0:
            raise MashmapError(MM_ESTATE, "no device-built index statistics in this context")
        mi = np.zeros(n, dtype=minmer_dtype)
        self._check(self._L.mm_index_download(self._h, _ptr(mi), None, None, None, None))
        return mi

    def tables_upload(self, sketch_cutoffs, min_hits):
        a = _c(sketch_cutoffs, np.int32)
        b = _c(min_hits, np.int32)
        self._check(self._L.mm_tables_upload(self._h, _ptr(a), len(a), _ptr(b), len(b)))

    def index_blob(self):
        p, n = C.c_void_p(), C.c_uint64()
        self._check(self._L.mm_index_blob(self._h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def index_blob_alloc(self, nbytes):
        p = C.c_void_p()
        self._check(self._L.mm_index_blob_alloc(self._h, nbytes, C.byref(p)))
        return p.value

    def index_adopt_blob(self):
        self._check(self._L.mm_index_adopt_blob(self._h))

    def sketch_segments(self, bases, segments):
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        segments = _c(segments, segment_dtype)
        out = np.zeros((len(segments), self.sketch_size), dtype=minmer_dtype)
        cnt = np.zeros(len(segments), dtype=np.int32)
        self._check(self._L.mm_sketch_segments(self._h, _ptr(bases), len(bases), _ptr(segments), len(segments),
                                               _ptr(out), _ptr(cnt)))
        return out, cnt

    def map_segments(self, bases, segments):
        """Returns (seg_results, candidates, loci) as numpy record arrays (host in, host out)."""
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        segments = _c(segments, segment_dtype)
        n = len(segments)
        self._n_segs = n
        seg_res = np.zeros(n, dtype=segres_dtype)
        cap_c, cap_l = 2 * n + 1024, 4 * n + 2048
        while True:
            cands = np.zeros(cap_c, dtype=l1_dtype)
            loci = np.zeros(cap_l, dtype=l2_dtype)
            nc, nl = C.c_uint64(), C.c_uint64()
            rc = self._L.mm_map_segments(self._h, _ptr(bases), len(bases), _ptr(segments), n, _ptr(seg_res),
                                         _ptr(cands), cap_c, C.byref(nc), _ptr(loci), cap_l, C.byref(nl))
            if rc == MM_ECAPACITY:
                cap_c, cap_l = max(cap_c, nc.value), max(cap_l, nl.value)
                continue
            self._check(rc)
            return seg_res, cands[: nc.value], loci[: nl.value]

    def batch_upload(self, bases, segments):
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        segments = _c(segments, segment_dtype)
        self._n_segs = len(segments)
        self._check(self._L.mm_batch_upload(self._h, _ptr(bases), len(bases), _ptr(segments), len(segments)))

    def batch_upload_packed(self, nibbles, n_bases, segments):
        """the batch as one nibble per base (see pack_bases): mm_batch_upload_packed"""
        nibbles = np.ascontiguousarray(nibbles, dtype=np.uint8)
        assert len(nibbles) >= (n_bases + 1) // 2
        segments = _c(segments, segment_dtype)
        self._n_segs = len(segments)
        self._check(self._L.mm_batch_upload_packed(self._h, _ptr(nibbles), int(n_bases), _ptr(segments), len(segments)))

    def map_segments_packed(self, nibbles, n_bases, segments):
        nibbles = np.ascontiguousarray(nibbles, dtype=np.uint8)
        segments = _c(segments, segment_dtype)
        n = len(segments)
        self._n_segs = n
        seg_res = np.zeros(n, dtype=segres_dtype)
        cand_cap, loci_cap = max(4 * n, 1024), max(8 * n, 2048)
        while True:
            cands = np.zeros(cand_cap, dtype=l1_dtype)
            loci = np.zeros(loci_cap, dtype=l2_dtype)
            nc, nl = C.c_uint64(), C.c_uint64()
            rc = self._L.mm_map_segments_packed(self._h, _ptr(nibbles), int(n_bases), _ptr(segments), n, _ptr(seg_res),
                                                _ptr(cands), cand_cap, C.byref(nc), _ptr(loci), loci_cap, C.byref(nl))
            if rc == MM_ECAPACITY:
                cand_cap, loci_cap = max(cand_cap, nc.value), max(loci_cap, nl.value)
                continue
            self._check(rc)
            self._nc, self._nl = nc.value, nl.value
            return seg_res, cands[: nc.value], loci[: nl.value]

    def pack_ms(self):
        v = C.c_float()
        self._L.mm_last_pack_ms(self._h, C.byref(v))
        return float(v.value)

    def map_resident(self):
        nc, nl = C.c_uint64(), C.c_uint64()
        self._check(self._L.mm_map_resident(self._h, C.byref(nc), C.byref(nl)))
        self._nc, self._nl = nc.value, nl.value
        return nc.value, nl.value

    def map_resident_l1_best(self):
        """phase 1 on a shard (mm_map_resident_l1_best): each segment's best intersection over this shard"""
        best = np.zeros(max(self._n_segs, 1), dtype=np.int32)
        self._check(self._L.mm_map_resident_l1_best(self._h, _ptr(best)))
        return best[: self._n_segs]

    def map_resident_with_best(self, best, points_after):
        """phase 2 (mm_map_resident_with_best): map with the best over all shards; points_after[seg]: a later shard has
        points of the segment"""
        b = _c(best, np.int32)
        a = _c(points_after, np.uint8)
        nc, nl = C.c_uint64(), C.c_uint64()
        self._check(self._L.mm_map_resident_with_best(self._h, _ptr(b), _ptr(a), C.byref(nc), C.byref(nl)))
        self._nc, self._nl = nc.value, nl.value
        return nc.value, nl.value

    def batch_fetch(self):
        seg_res = np.zeros(self._n_segs, dtype=segres_dtype)
        cands = np.zeros(max(self._nc, 1), dtype=l1_dtype)
        loci = np.zeros(max(self._nl, 1), dtype=l2_dtype)
        self._check(self._L.mm_batch_fetch(self._h, _ptr(seg_res), _ptr(cands), len(cands), _ptr(loci), len(loci)))
        return seg_res, cands[: self._nc], loci[: self._nl]

    def batch_fetch_sketch(self):
        out = np.zeros((self._n_segs, self.sketch_size), dtype=minmer_dtype)
        cnt = np.zeros(self._n_segs, dtype=np.int32)
        self._check(self._L.mm_batch_fetch_sketch(self._h, _ptr(out), _ptr(cnt)))
        return out, cnt

    def stage_ms(self):
        arr = (C.c_float * 8)()
        self._L.mm_last_stage_ms(self._h, C.byref(arr))
        return list(arr)


# ---- include/mashmap_b200_align.h (base-level alignment of mappings, in the same library) ----------------------------

align_job_dtype = np.dtype([("q_offset", "<u8"), ("t_offset", "<u8"), ("q_len", "<i4"), ("t_len", "<i4"), ("k", "<i4"),
                            ("mode", "<i4")])
MM_ALIGN_HW, MM_ALIGN_NW = 0, 1  # align_job_dtype["mode"]: edlib's EDLIB_MODE_HW / EDLIB_MODE_NW
MM_ALIGN_BAND_MIN_LEN = 32 * 1024  # NW sub-problems with max(q_len, t_len) >= this run banded, one CTA per sweep
align_result_dtype = np.dtype([("ed", "<i4"), ("start", "<i4"), ("end", "<i4"), ("alignment_length", "<i4"),
                               ("ops_offset", "<u8")])
align_tag_result_dtype = np.dtype([("ed", "<i4"), ("alignment_length", "<i4"), ("cg_offset", "<u8"), ("cg_len", "<u8"),
                                   ("cs_offset", "<u8"), ("cs_len", "<u8")])
MM_ALIGN_TAG_EQX, MM_ALIGN_TAG_CS = 1, 2  # flags of mm_align_batch_tags: extended CIGAR (= / X), minimap2's short cs
assert align_job_dtype.itemsize == 32 and align_result_dtype.itemsize == 24 and align_tag_result_dtype.itemsize == 40

ALIGN_EXPORTED_SYMBOLS = ["mm_align_ctx_create", "mm_align_ctx_destroy", "mm_align_last_error", "mm_align_batch",
                          "mm_align_last_stage_ms", "mm_align_batch_tags", "mm_align_last_tag_ms"]


def _align_lib():
    L = lib()
    if not getattr(L, "_align_bound", False):
        vp, u64 = C.c_void_p, C.c_uint64
        L.mm_align_ctx_create.argtypes = [C.c_int, u64, C.POINTER(vp)]
        L.mm_align_ctx_destroy.argtypes = [vp]
        L.mm_align_last_error.argtypes = [vp]
        L.mm_align_last_error.restype = C.c_char_p
        L.mm_align_batch.argtypes = [vp, vp, u64, vp, u64, vp, u64, vp, vp, u64, C.POINTER(u64)]
        L.mm_align_last_stage_ms.argtypes = [vp, C.POINTER(C.c_float * 8)]
        L.mm_align_batch_tags.argtypes = [vp, vp, u64, vp, u64, vp, u64, C.c_uint32, vp, vp, u64, C.POINTER(u64)]
        L.mm_align_last_tag_ms.argtypes = [vp, C.POINTER(C.c_float)]
        L._align_bound = True
    return L


class AlignContext:
    """mm_align_ctx: edlibAlign(HW or NW, PATH) for batches of (query, target, k, mode) on one device."""

    def __init__(self, device=0, scratch_bytes=0):
        L = _align_lib()
        self._ctx = C.c_void_p()
        rc = L.mm_align_ctx_create(int(device), int(scratch_bytes), C.byref(self._ctx))
        if rc != MM_OK:
            raise MashmapError(rc, L.mm_align_last_error(None).decode())

    def align(self, qbases, tbases, jobs, ops_cap=None):
        """jobs: align_job_dtype array. Returns (results, ops) with ops the concatenated edit ops (0 M, 1 I, 2 D, 3 X)."""
        L = _align_lib()
        q = np.ascontiguousarray(qbases, dtype=np.uint8)
        t = np.ascontiguousarray(tbases, dtype=np.uint8)
        jobs = np.ascontiguousarray(jobs, dtype=align_job_dtype)
        res = np.zeros(len(jobs), dtype=align_result_dtype)
        if ops_cap is None:
            ops_cap = int(jobs["q_len"].astype(np.int64).sum() + jobs["t_len"].astype(np.int64).sum())
        ops = np.zeros(max(int(ops_cap), 1), dtype=np.uint8)
        n = C.c_uint64()
        rc = L.mm_align_batch(self._ctx, _ptr(q), len(q), _ptr(t), len(t), _ptr(jobs), len(jobs), _ptr(res), _ptr(ops),
                              int(ops_cap), C.byref(n))
        if rc != MM_OK:
            err = MashmapError(rc, L.mm_align_last_error(self._ctx).decode())
            err.n_ops = n.value
            raise err
        return res, ops[: n.value]

    def align_tags(self, qbases, tbases, jobs, flags=0, text_cap=None):
        """mm_align_batch_tags: jobs (MM_ALIGN_NW only) as for align(). Returns (results, text) with results an
        align_tag_result_dtype array and text the bytes its cg / cs offsets point into. On MM_ECAPACITY the raised error
        carries n_text, the size needed."""
        L = _align_lib()
        q = np.ascontiguousarray(qbases, dtype=np.uint8)
        t = np.ascontiguousarray(tbases, dtype=np.uint8)
        jobs = np.ascontiguousarray(jobs, dtype=align_job_dtype)
        res = np.zeros(len(jobs), dtype=align_tag_result_dtype)
        if text_cap is None:  # a run of L ops takes at most 2L bytes of cg and 3L of cs; a path is at most Q + T ops
            ops = int(jobs["q_len"].astype(np.int64).sum() + jobs["t_len"].astype(np.int64).sum())
            text_cap = ops * (5 if flags & MM_ALIGN_TAG_CS else 2)
        text = np.zeros(max(int(text_cap), 1), dtype=np.uint8)
        n = C.c_uint64()
        rc = L.mm_align_batch_tags(self._ctx, _ptr(q), len(q), _ptr(t), len(t), _ptr(jobs), len(jobs), int(flags),
                                   _ptr(res), _ptr(text), int(text_cap), C.byref(n))
        if rc != MM_OK:
            err = MashmapError(rc, L.mm_align_last_error(self._ctx).decode())
            err.n_text = n.value
            raise err
        return res, text[: n.value].tobytes()

    def stage_ms(self):
        a = (C.c_float * 8)()
        _align_lib().mm_align_last_stage_ms(self._ctx, C.byref(a))
        return list(a)

    def tag_ms(self):
        """the formatting kernels' time of the last align_tags, in ms"""
        a = C.c_float()
        _align_lib().mm_align_last_tag_ms(self._ctx, C.byref(a))
        return a.value

    def close(self):
        if self._ctx:
            _align_lib().mm_align_ctx_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
