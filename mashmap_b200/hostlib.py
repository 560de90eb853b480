"""ctypes view of the host-side C++ (libmashmap_host.so: skch::Stat, the host index builder, the host
tail) for tests and bench.py. The mapping itself is only reachable through capi (the CUDA library)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import capi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmashmap_host.so")
CLI_PATH = os.path.join(_HERE, "mashmap-b200")


class TailParams(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "kmerSize", "segLength", "sketchSize", "filterMode", "numMappingsForSegment", "numMappingsForShortSequence",
        "block_length", "chain_gap", "mergeMappings", "stage1_topANI_filter", "keep_low_pct_id", "skip_self",
        "skip_prefix", "prefix_delim", "filterLengthMismatches", "legacy_output", "report_ANI_percentage")] + [
        (n, C.c_float) for n in ("percentageIdentity", "ANIDiff", "ANIDiffConf", "kmerComplexityThreshold")]


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} not built: run __graft_entry__.build()")
        capi.lib()  # dependency (same directory, rpath $ORIGIN)
        L = C.CDLL(LIB_PATH)
        L.skch_binomial_Q.argtypes = [C.c_uint, C.c_double, C.c_uint]
        L.skch_binomial_Q.restype = C.c_double
        L.skch_j2md.argtypes = [C.c_float, C.c_int]
        L.skch_j2md.restype = C.c_float
        L.skch_md2j.argtypes = [C.c_float, C.c_int]
        L.skch_md2j.restype = C.c_float
        L.skch_md_lower_bound.argtypes = [C.c_float, C.c_int, C.c_int]
        L.skch_md_lower_bound.restype = C.c_float
        L.skch_min_hits.argtypes = [C.c_int, C.c_int, C.c_float]
        L.skch_recommended_sketch_size.argtypes = [C.c_int, C.c_float, C.c_int64, C.c_uint64]
        L.skch_recommended_sketch_size.restype = C.c_int64
        L.skch_sketch_cutoffs.argtypes = [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int, C.c_void_p, C.c_int]
        L.skch_add_minmers.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64]
        L.skch_add_minmers.restype = C.c_int64
        L.skch_tail_create.argtypes = [C.POINTER(TailParams), C.c_int, C.POINTER(C.c_char_p), C.c_void_p, C.c_void_p]
        L.skch_tail_create.restype = C.c_void_p
        L.skch_tail_destroy.argtypes = [C.c_void_p]
        L.skch_tail_map_read.argtypes = [C.c_void_p, C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                         C.c_uint32, C.c_void_p, C.c_void_p, C.POINTER(C.c_int32)]
        L.skch_tail_map_read.restype = C.c_char_p
        L.skch_fasta_readers_diff.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.skch_fasta_readers_diff.restype = C.c_int64
        L.skch_mmi_inflate.argtypes = [C.c_char_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint32)]
        L.skch_bgzf_error.restype = C.c_char_p
        L.skch_bgzf_text.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_int64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                     C.POINTER(C.c_uint64)]
        L.skch_bgzf_text.restype = C.c_int64
        L.skch_gzread_text.argtypes = [C.c_char_p, C.c_void_p, C.c_uint64]
        L.skch_gzread_text.restype = C.c_int64
        L.skch_bgzf_readers_diff.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
        L.skch_bgzf_readers_diff.restype = C.c_int64
        L.skch_bgzf_read_digest.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                            C.POINTER(C.c_uint64)]
        L.skch_fastq_error.restype = C.c_char_p
        L.skch_fastq_digest.argtypes = [C.c_char_p, C.c_uint64, C.c_int, C.c_int, C.POINTER(C.c_uint64 * 4)]
        L.skch_index_from_minmers.argtypes = [C.c_void_p, C.c_uint64, C.c_int, C.c_float]
        L.skch_index_from_minmers.restype = C.c_void_p
        L.skch_index_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float]
        L.skch_index_build.restype = C.c_void_p
        L.skch_index_from_cli.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
        L.skch_index_from_cli.restype = C.c_void_p
        L.skch_params_from_cli.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
        L.skch_params_from_cli.restype = C.c_void_p
        L.skch_index_params.argtypes = [C.c_void_p, C.c_void_p]
        L.skch_index_metadata_only.argtypes = [C.c_int] * 5
        L.skch_index_metadata_only.restype = C.c_void_p
        L.skch_index_destroy.argtypes = [C.c_void_p]
        L.skch_index_sizes.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                       C.POINTER(C.c_int32)]
        L.skch_index_copy.argtypes = [C.c_void_p] * 6
        L.skch_index_upload.argtypes = [C.c_void_p, C.c_void_p]
        vp = C.c_void_p
        L.skch_bm_create.argtypes = [vp, C.c_float, C.c_int, C.c_int]
        L.skch_bm_create.restype = vp
        L.skch_bm_create_ex.argtypes = [vp, C.c_float, C.c_int, C.c_int, C.c_int, vp, C.c_int]
        L.skch_bm_create_ex.restype = vp
        L.skch_mapping_record_bytes.restype = C.c_uint32
        L.skch_bm_results_raw.argtypes = [vp, vp, C.c_uint64]
        L.skch_bm_results_raw.restype = C.c_uint64
        L.skch_bm_one_to_one.argtypes = [vp, vp, C.c_uint64, C.c_int32, C.c_int32]
        L.skch_bm_one_to_one.restype = C.c_uint64
        L.skch_bm_paf_final.argtypes = [vp, C.POINTER(C.c_uint64)]
        L.skch_bm_paf_final.restype = vp
        L.skch_bm_device_count.argtypes = [vp]
        L.skch_bm_destroy.argtypes = [vp]
        L.skch_bm_ctx.argtypes = [vp]
        L.skch_bm_ctx.restype = vp
        L.skch_bm_batch_create.argtypes = [vp, C.c_uint64, C.c_int32, C.c_int32]
        L.skch_bm_batch_create.restype = vp
        L.skch_bm_batch_fill.argtypes = [vp, vp, C.c_int]
        L.skch_bm_batch_fill.restype = C.c_double
        L.skch_bm_batch_bytes.argtypes = [vp]
        L.skch_bm_batch_bytes.restype = C.c_uint64
        L.skch_pack_bases.argtypes = [vp, C.c_uint64, vp]
        L.skch_bm_batch_segments.argtypes = [vp, C.POINTER(vp)]
        L.skch_bm_batch_segments.restype = C.c_uint64
        L.skch_bm_batch_destroy.argtypes = [vp]
        L.skch_bm_map.argtypes = [vp, vp, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                  C.POINTER(C.c_float * 8), C.POINTER(C.c_double), C.POINTER(C.c_double)]
        L.skch_bm_paf.argtypes = [vp, C.POINTER(C.c_uint64)]
        L.skch_bm_paf.restype = vp
        L.skch_bm_results.argtypes = [vp, vp, C.c_uint64]
        L.skch_bm_results.restype = C.c_uint64
        L.skch_plan_shards.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp]
        L.skch_last_plan_error.restype = C.c_char_p
        L.skch_global_frequent_seeds.argtypes = [C.c_int, vp, vp, vp, C.c_float, vp, C.c_uint64, C.POINTER(C.c_int32),
                                                 C.POINTER(C.c_uint64)]
        L.skch_global_frequent_seeds.restype = C.c_int64
        _lib = L
    return _lib


class BatchMapper:
    """skch::BatchMapper: reads in pinned host memory -> one device call -> host tail -> PAF text."""

    FILTER_MODES = {"map": 1, "one-to-one": 2, "none": 3}

    def __init__(self, host_index, pi=0.85, device=0, threads=8, filter_mode="map", devices=None):
        """devices: several GPUs driven by this one process (skch::Map --devices); the index image is replicated with
        one grouped NCCL broadcast and the parts of every batch are dealt to the devices round robin"""
        self.index = host_index
        devs = np.ascontiguousarray(devices if devices else [], dtype=np.int32)
        self.h = lib().skch_bm_create_ex(host_index.h, pi, device, threads, self.FILTER_MODES[filter_mode],
                                         devs.ctypes.data if len(devs) else None, len(devs))
        self.ctx_handle = lib().skch_bm_ctx(self.h)
        self.record_bytes = int(lib().skch_mapping_record_bytes())

    def results_raw(self):
        """the mappings of the last map() as raw skch::MappingResult records ([n, record_bytes] uint8): what a rank hands
        to mm_records_allgather"""
        n = lib().skch_bm_results_raw(self.h, None, 0)
        need = max(n, 1) * self.record_bytes
        buf = getattr(self, "_raw_pin", None)
        if buf is None or buf.nbytes < need:  # a pinned buffer kept between calls: the records go to the device next
            self._raw_pin = buf = capi.PinnedBuffer(need + need // 4)
        out = buf.array[:need].reshape(max(n, 1), self.record_bytes)
        lib().skch_bm_results_raw(self.h, out.ctypes.data, n)
        return out[:n]

    def one_to_one(self, records, n_queries, query_len, copy=True):
        """-f one-to-one, the run-wide step over raw records of any origin (this rank's, or all ranks' after the all-gather):
        returns (mappings kept, PAF text). copy=False hands back a view of the text where the library wrote it (valid until
        the next call) instead of a Python copy of it"""
        r = np.ascontiguousarray(records, dtype=np.uint8)
        kept = lib().skch_bm_one_to_one(self.h, r.ctypes.data, len(r), int(n_queries), int(query_len))
        return int(kept), self.paf_final(copy)

    def paf_final(self, copy=True):
        """the PAF text of the last one_to_one()"""
        n = C.c_uint64()
        p = lib().skch_bm_paf_final(self.h, C.byref(n))
        if copy:
            return C.string_at(p, n.value)
        return memoryview((C.c_char * n.value).from_address(C.cast(p, C.c_void_p).value)) if n.value else memoryview(b"")

    @property
    def device_count(self):
        return int(lib().skch_bm_device_count(self.h))

    def make_batch(self, n_reads, read_len, first_seq_counter=0):
        return ReadBatch(self, n_reads, read_len, first_seq_counter)

    def map(self, batch):
        pb, nr, nm = C.c_uint64(), C.c_uint64(), C.c_uint64()
        ms = (C.c_float * 8)()
        sd, st = C.c_double(), C.c_double()
        lib().skch_bm_map(self.h, batch.h, C.byref(pb), C.byref(nr), C.byref(nm), C.byref(ms), C.byref(sd), C.byref(st))
        return dict(paf_bytes=pb.value, mapped_reads=nr.value, mappings=nm.value, stage_ms=list(ms), sec_device=sd.value,
                    sec_tail=st.value)

    def paf(self):
        n = C.c_uint64()
        p = lib().skch_bm_paf(self.h, C.byref(n))
        return C.string_at(p, n.value).decode()

    def results(self):
        n = lib().skch_bm_results(self.h, None, 0)
        out = np.zeros((max(n, 1), 10), dtype=np.int32)
        lib().skch_bm_results(self.h, out.ctypes.data, n)
        return out[:n]

    def close(self):
        if self.h:
            lib().skch_bm_destroy(self.h)
            self.h = None


class ReadBatch:
    def __init__(self, bm, n_reads, read_len, first_seq_counter):
        self.h = lib().skch_bm_batch_create(bm.h, n_reads, read_len, first_seq_counter)
        self.n_reads, self.read_len = n_reads, read_len
        sp = C.c_void_p()
        ns = lib().skch_bm_batch_segments(self.h, C.byref(sp))
        buf = (C.c_char * (ns * capi.segment_dtype.itemsize)).from_address(sp.value)
        self.segments = np.frombuffer(buf, dtype=capi.segment_dtype, count=ns)

    def fill(self, ascii_reads, threads=8):
        """packs the reads (text, read r at r * read_len) into the pinned batch buffer as nibbles -- what the FASTA
        reader of skch::Map does while it parses. Returns the seconds the packing took."""
        a = np.ascontiguousarray(ascii_reads, dtype=np.uint8).reshape(-1)
        assert len(a) == self.n_reads * self.read_len
        return float(lib().skch_bm_batch_fill(self.h, a.ctypes.data, int(threads)))

    @property
    def h2d_bytes(self):
        """bytes of bases that cross PCIe per mapping pass"""
        return int(lib().skch_bm_batch_bytes(self.h))

    def close(self):
        if self.h:
            lib().skch_bm_batch_destroy(self.h)
            self.h = None


def pack_bases(ascii_bases):
    """the host library's packer (seqio::pack_bases, AVX2): text -> one nibble per base"""
    a = np.ascontiguousarray(ascii_bases, dtype=np.uint8)
    out = np.zeros((len(a) + 1) // 2, dtype=np.uint8)
    lib().skch_pack_bases(a.ctypes.data, len(a), out.ctypes.data)
    return out


class HostIndex:
    """skch::Sketch built by the host library (from sequences in memory, or from an existing minmer list)."""

    def __init__(self, handle):
        self.h = handle
        a, b, c, t = C.c_uint64(), C.c_uint64(), C.c_uint64(), C.c_int32()
        lib().skch_index_sizes(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(t))
        self.n_minmers, self.n_keys, self.n_points, self.freq_threshold = a.value, b.value, c.value, t.value

    @classmethod
    def build(cls, seqs, offs, k, seg_length, sketch_size, threads=8, kmer_pct_threshold=0.001):
        seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
        offs = np.ascontiguousarray(offs, dtype=np.uint64)
        h = lib().skch_index_build(seqs.ctypes.data, offs.ctypes.data, len(offs) - 1, k, seg_length, sketch_size, threads,
                                   kmer_pct_threshold)
        return cls(h)

    @classmethod
    def metadata_only(cls, n_contigs, contig_len, k, seg_length, sketch_size):
        return cls(lib().skch_index_metadata_only(n_contigs, contig_len, k, seg_length, sketch_size))

    @classmethod
    def from_cli(cls, args):
        """skch::Sketch built the way the driver program does it, from the reference's command-line options
        (FASTA files, --saveIndex / --loadIndex ...). Host only."""
        argv = (C.c_char_p * len(args))(*[a.encode() for a in args])
        return cls(lib().skch_index_from_cli(len(args), argv))

    @classmethod
    def params_from_cli(cls, args):
        """command line -> skch::Parameters only (no Sketch is built, the reference file is not read)"""
        argv = (C.c_char_p * len(args))(*[a.encode() for a in args])
        return cls(lib().skch_params_from_cli(len(args), argv))

    def params_into(self, struct):
        """fills a ctypes structure laid out like tests/refh.py::OrcParams with the parsed skch::Parameters"""
        lib().skch_index_params(self.h, C.byref(struct))
        return struct

    @classmethod
    def from_minmers(cls, minmers, n_contigs, kmer_pct_threshold=0.001):
        m = np.ascontiguousarray(minmers, dtype=capi.minmer_dtype)
        return cls(lib().skch_index_from_minmers(m.ctypes.data, len(m), n_contigs, kmer_pct_threshold))

    def arrays(self):
        mi = np.zeros(self.n_minmers, dtype=capi.minmer_dtype)
        keys = np.zeros(self.n_keys, dtype=np.uint64)
        offs = np.zeros(self.n_keys + 1, dtype=np.uint64)
        pts = np.zeros(self.n_points, dtype=capi.ipoint_dtype)
        fr = np.zeros(self.n_keys, dtype=np.uint8)
        lib().skch_index_copy(self.h, mi.ctypes.data, keys.ctypes.data, offs.ctypes.data, pts.ctypes.data, fr.ctypes.data)
        return mi, keys, offs, pts, fr

    def upload(self, ctx):
        rc = lib().skch_index_upload(self.h, ctx._h)
        ctx._check(rc)

    def close(self):
        if self.h:
            lib().skch_index_destroy(self.h)
            self.h = None


def fasta_readers_diff(path, threads=4):
    """(differences, records, bases): the mapped bulk FASTA reader against the line reader; differences = -1 if the bulk
    reader declines the file (gzip, FASTQ ...)"""
    nr, nb = C.c_uint64(), C.c_uint64()
    d = lib().skch_fasta_readers_diff(path.encode(), threads, C.byref(nr), C.byref(nb))
    return d, nr.value, nb.value


def mmi_inflate(comp, out_len):
    """the host build of mm_inflate.h on one raw DEFLATE stream that must inflate to exactly out_len bytes:
    (mmi_status, text, CRC-32)"""
    comp = bytes(comp)
    out = np.zeros(max(int(out_len), 1), dtype=np.uint8)
    crc = C.c_uint32()
    rc = lib().skch_mmi_inflate(comp, len(comp), out.ctypes.data_as(C.c_void_p), int(out_len), C.byref(crc))
    return rc, out[: int(out_len)].tobytes(), crc.value


def bgzf_text(path, window_bytes=1 << 20, threads=2, fail_block=-1):
    """(text, windows, inflater calls) as the windowed BGZF reader hands the text over (host inflater); text is None if
    the reader declines the file; raises RuntimeError with the reader's message on an error"""
    nw, nc = C.c_uint64(), C.c_uint64()
    n = lib().skch_bgzf_text(path.encode(), window_bytes, threads, fail_block, None, 0, C.byref(nw), C.byref(nc))
    if n == -1:
        return None, 0, 0
    if n < 0:
        raise RuntimeError(lib().skch_bgzf_error().decode())
    buf = np.zeros(max(n, 1), dtype=np.uint8)
    lib().skch_bgzf_text(path.encode(), window_bytes, threads, fail_block, buf.ctypes.data_as(C.c_void_p), n, C.byref(nw), C.byref(nc))
    return buf[:n].tobytes(), nw.value, nc.value


def gzread_text(path):
    """everything zlib's gzread gives for the file: the text the line reader reads"""
    n = lib().skch_gzread_text(path.encode(), None, 0)
    buf = np.zeros(max(n, 1), dtype=np.uint8)
    lib().skch_gzread_text(path.encode(), buf.ctypes.data_as(C.c_void_p), n)
    return buf[:n].tobytes()


def fastq_digest(path, window_bytes=0, threads=2, device=-1):
    """(records, bases, digest, windows) of a file's records (name, length, nibbles): the line reader (window_bytes = 0),
    or the FASTQ window reader with the host build of mm_fastq.h (device < 0) or mm_fastq on that device. None if the
    window reader declines the file; RuntimeError on a read error."""
    out = (C.c_uint64 * 4)()
    rc = lib().skch_fastq_digest(path.encode(), int(window_bytes), threads, device, C.byref(out))
    if rc == -1:
        return None
    if rc != 0:
        raise RuntimeError(lib().skch_fastq_error().decode() if rc == -3 else f"cannot read {path}")
    return tuple(int(x) for x in out)


def bgzf_readers_diff(path, window_bytes, threads=2):
    """(differences, records, bases): the windowed BGZF reader (host inflater) against the line reader; -1 if it
    declines the file"""
    nr, nb = C.c_uint64(), C.c_uint64()
    d = lib().skch_bgzf_readers_diff(path.encode(), window_bytes, threads, C.byref(nr), C.byref(nb))
    return d, nr.value, nb.value


def lookup_from_minmers(minmers, n_contigs, kmer_pct_threshold=0.001):
    """Sketch::index + frequency filter: (minmers after dropFreqSeedSet, keys, offsets, points, is_freq)"""
    hi = HostIndex.from_minmers(minmers, n_contigs, kmer_pct_threshold)
    out = hi.arrays()
    hi.close()
    return out


def add_minmers_chunked(seq, k, w, s, chunk, warm, seq_id=0):
    """CommonFunc::addMinmersChunked: the chunked + stitched window scan of the GPU index builder, run on the host.
    Returns (records, number of chunks that were re-scanned from the previous chunk's exact state)"""
    b = seq.tobytes() if isinstance(seq, np.ndarray) else bytes(seq)
    L = lib()
    L.skch_add_minmers_chunked.restype = C.c_int64
    L.skch_add_minmers_chunked.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int64,
                                           C.c_void_p, C.c_int64, C.POINTER(C.c_int32)]
    cap = 2 * len(b) + 1024
    out = np.zeros(cap, dtype=capi.minmer_dtype)
    r = C.c_int32()
    n = L.skch_add_minmers_chunked(b, len(b), k, w, s, seq_id, chunk, warm, out.ctypes.data, cap, C.byref(r))
    return out[:n].copy(), int(r.value)


def min_hits_table(sketch_size, k, pi):
    L = lib()
    return np.array([0] + [L.skch_min_hits(s, k, pi) for s in range(1, sketch_size + 1)], dtype=np.int32)


def sketch_cutoffs(sketch_size, k, ani_diff=0.0, ani_diff_conf=0.999, enabled=True):
    out = np.zeros(1002, dtype=np.int32)
    n = lib().skch_sketch_cutoffs(sketch_size, k, ani_diff, ani_diff_conf, int(enabled), out.ctypes.data, len(out))
    return out[:n].copy()


def add_minmers(seq, k, w, s, seq_id=0, stable_ties=False):
    """CommonFunc::addMinmers of one contig on the host. stable_ties: records with equal (wpos, wpos_end) stay in emission
    order (what the GPU builder does) instead of the order std::sort happens to leave them in (what the reference does)"""
    b = seq.tobytes() if isinstance(seq, np.ndarray) else bytes(seq)
    cap = max(1024, 4 * (len(b) // max(1, w) + 2) * (s + 2) + 4 * len(b) // 10)
    L = lib()
    L.skch_add_minmers_ex.restype = C.c_int64
    L.skch_add_minmers_ex.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.c_int]
    while True:
        out = np.zeros(cap, dtype=capi.minmer_dtype)
        n = L.skch_add_minmers_ex(b, len(b), k, w, s, seq_id, out.ctypes.data, cap, 1 if stable_ties else 0)
        if n >= 0:
            return out[:n].copy()
        cap = -n + 16


class HostTail:
    def __init__(self, tp: TailParams, names, lens, groups=None):
        L = lib()
        arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
        self._lens = np.ascontiguousarray(lens, dtype=np.int32)
        self._groups = None if groups is None else np.ascontiguousarray(groups, dtype=np.int32)
        self.h = L.skch_tail_create(C.byref(tp), len(names), arr, self._lens.ctypes.data,
                                    None if self._groups is None else self._groups.ctypes.data)

    def map_read(self, name, length, seq_counter, segs, seg_res, cands, loci, ref_group=-1):
        segs = np.ascontiguousarray(segs, dtype=capi.segment_dtype)
        seg_res = np.ascontiguousarray(seg_res, dtype=capi.segres_dtype)
        cands = np.ascontiguousarray(cands, dtype=capi.l1_dtype)
        loci = np.ascontiguousarray(loci, dtype=capi.l2_dtype)
        n = C.c_int32()
        txt = lib().skch_tail_map_read(self.h, name.encode(), length, seq_counter, ref_group, segs.ctypes.data,
                                       seg_res.ctypes.data, len(segs), cands.ctypes.data if len(cands) else None,
                                       loci.ctypes.data if len(loci) else None, C.byref(n))
        return txt.decode(), n.value

    def close(self):
        if self.h:
            lib().skch_tail_destroy(self.h)
            self.h = None


def plan_shards(contig_len, groups, by_group, n_shards):
    """--indexShards' plan (skch::BatchMapper::planShards): the first contig of every shard plus the contig count, or
    ValueError with the reason the reference cannot be cut so"""
    ln = np.ascontiguousarray(contig_len, dtype=np.uint64)
    gr = np.ascontiguousarray(groups, dtype=np.int32)
    first = np.zeros(max(n_shards, 0) + 1, dtype=np.int32)
    if lib().skch_plan_shards(ln.ctypes.data, gr.ctypes.data, len(ln), int(by_group), n_shards, first.ctypes.data) != 0:
        raise ValueError(lib().skch_last_plan_error().decode())
    return first


def global_frequent_seeds(shard_keys, shard_counts, kmer_pct_threshold):
    """the frequent seeds of a reference indexed in shards, from each shard's distinct hashes (ascending) and their
    interval-point counts: (threshold, number of distinct hashes, frequent hashes ascending)"""
    ks = [np.ascontiguousarray(k, dtype=np.uint64) for k in shard_keys]
    cs = [np.ascontiguousarray(c, dtype=np.uint32) for c in shard_counts]
    kp = (C.c_void_p * len(ks))(*[k.ctypes.data for k in ks])
    cp = (C.c_void_p * len(cs))(*[c.ctypes.data for c in cs])
    n = np.array([len(k) for k in ks], dtype=np.uint64)
    out = np.zeros(max(1, int(n.sum())), dtype=np.uint64)
    thr, uniq = C.c_int32(0), C.c_uint64(0)
    m = lib().skch_global_frequent_seeds(len(ks), C.cast(kp, C.c_void_p), C.cast(cp, C.c_void_p), n.ctypes.data,
                                         kmer_pct_threshold, out.ctypes.data, len(out), C.byref(thr), C.byref(uniq))
    assert m >= 0
    return int(thr.value), int(uniq.value), out[:m].copy()
