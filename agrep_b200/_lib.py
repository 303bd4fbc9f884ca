"""ctypes view of libagrepb200.so (include/agrep_b200.h).  The library is the product; this module only
declares its C ABI for Python callers (tests, bench.py).  No computation happens in Python."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libagrepb200.so")

AGB_MAXERR, AGB_MAXDELIM, AGB_MAXANCHOR = 8, 8, 24
WANT_COUNT, WANT_RECORDS, WANT_ORDINALS, WANT_LEVELS = 0, 1, 2, 4
PLAN_ALL, PLAN_ANCHORS = 0, 1
ENGINE_NAMES = {0: "bitap", 1: "asearch", 2: "asearch0", 3: "asearch1", 4: "sgrep_bm", 5: "regex"}
ENGINE_REGEX = 5
REGEX_MAXPOS = 63
WIDE_WORDS = 5
WIDE_MAXPOS = 64 * WIDE_WORDS - 1


class Options(C.Structure):
    _fields_ = [("k", C.c_int32), ("nocase", C.c_int32), ("wordbound", C.c_int32), ("wholeline", C.c_int32),
                ("inverse", C.c_int32), ("linenum", C.c_int32), ("ins_free", C.c_int32),
                ("cost_i", C.c_int32), ("cost_s", C.c_int32), ("cost_d", C.c_int32),
                ("bestmatch", C.c_int32), ("regex", C.c_int32), ("delim", C.c_char_p), ("wide_approx", C.c_int32),
                ("sticky_delim", C.c_int32)]


class Desc(C.Structure):
    _fields_ = [("mask", C.c_uint64 * 256),
                ("init0", C.c_uint64), ("init1", C.c_uint64), ("noerr", C.c_uint64), ("endpos", C.c_uint64),
                ("dendpos", C.c_uint64), ("dmask", C.c_uint64), ("wildmask", C.c_uint64),
                ("reset", C.c_uint64 * (2 * AGB_MAXERR + 1)), ("start", C.c_uint64 * (2 * AGB_MAXERR + 1)),
                ("start_closes", C.c_int32), ("M", C.c_int32), ("L", C.c_int32),
                ("delim", C.c_uint8 * (2 * AGB_MAXDELIM + 2)),
                ("delim_kind", C.c_int32), ("k", C.c_int32), ("nrows", C.c_int32),
                ("cost_i", C.c_int32), ("cost_s", C.c_int32), ("cost_d", C.c_int32),
                ("engine", C.c_int32), ("and_mode", C.c_int32), ("inverse", C.c_int32),
                ("user_delim", C.c_int32), ("outtail", C.c_int32),
                ("plan", C.c_int32), ("n_anchors", C.c_int32), ("anchor_len", C.c_int32),
                ("anchor", C.c_uint32 * AGB_MAXANCHOR), ("anchor_fold", C.c_uint32), ("anchor_mask", C.c_uint32),
                ("refine", C.c_int32), ("pat_len", C.c_int32), ("anchor_off", C.c_int32 * AGB_MAXANCHOR),
                ("n_anchors3", C.c_int32), ("anchor3", C.c_uint32 * 4), ("anchor3_off", C.c_int32 * 4), ("adaptive", C.c_int32),
                ("delim_fold", C.c_uint8 * (2 * AGB_MAXDELIM + 2)), ("pair_plan", C.c_uint8), ("wide", C.c_uint8),
                ("sticky_delim", C.c_uint8)]


class Regex(C.Structure):
    _fields_ = [("follow", C.c_uint64 * (REGEX_MAXPOS + 1)), ("head", C.c_int32), ("tail", C.c_int32), ("pad", C.c_int32 * 2)]


class Wide(C.Structure):
    _W = C.c_uint64 * WIDE_WORDS
    _fields_ = [("mask", _W * 256), ("init0", _W), ("init1", _W), ("noerr", _W), ("endpos", _W),
                ("dendpos", _W), ("dmask", _W), ("reset", _W), ("start", _W),
                ("reset_up", _W * AGB_MAXERR), ("start_up", _W * AGB_MAXERR)]


class Record(C.Structure):
    _fields_ = [("begin", C.c_int64), ("end", C.c_int64), ("ordinal", C.c_int64), ("level", C.c_int32), ("pad", C.c_int32)]


class Result(C.Structure):
    _fields_ = [("n_matched", C.c_uint64), ("n_records", C.c_uint64), ("n_flagged", C.c_uint64),
                ("level_hist", C.c_uint64 * (AGB_MAXERR + 1)), ("ms_front", C.c_float), ("ms_records", C.c_float),
                ("n_closes", C.c_uint64), ("truncated", C.c_uint32), ("pad", C.c_uint32)]


class CorpusSpec(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_bytes", C.c_uint64), ("first_page", C.c_uint64),
                ("paragraphs", C.c_int32), ("needle_every", C.c_int32), ("needle", C.c_char * 64),
                ("needle_maxedits", C.c_int32), ("pad", C.c_int32)]


EXPORTS = ["agb_fill_ordinals", "agb_compile", "agb_pattern_free", "agb_pattern_desc", "agb_pattern_from_desc", "agb_scan_device",
           "agb_pattern_regex", "agb_pattern_from_regex", "agb_pattern_wide",
           "agb_scan_host", "agb_scan_fd", "agb_scan_host_windowed", "agb_scan_fd_windowed", "agb_scan_set", "agb_bestmatch_device", "agb_corpus_fill_device", "agb_corpus_fill_host",
           "agb_last_error", "agb_device_count", "agb_set_device", "agb_version", "agb_kernel_launches", "agb_shutdown",
           "agb_text_from_host", "agb_text_from_fd", "agb_text_free", "agb_text_size", "agb_text_device", "agb_scan_text",
           "agb_comm_unique_id", "agb_comm_init", "agb_comm_free", "agb_comm_world", "agb_comm_rank", "agb_shard_halo",
           "agb_scan_sharded", "agb_scan_shard_local", "agb_bestmatch_sharded"]

HALO_LEFT, HALO_RIGHT = 512, 65536


class ShardPart(C.Structure):
    _fields_ = [("closes", C.c_uint64), ("ord_fix", C.c_int64), ("ord_origin", C.c_int64), ("byte_base", C.c_int64),
                ("virt", C.c_int32), ("pad", C.c_int32)]

_lib = None


def lib():
    """Loads the CUDA library; raises if it is missing -- there is no fallback implementation."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libagrepb200.so is not built: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(or make -C agrep_b200/csrc); there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.agb_compile.argtypes = [C.c_char_p, C.POINTER(Options), C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.agb_compile.restype = C.c_int
    L.agb_pattern_free.argtypes = [C.c_void_p]
    L.agb_pattern_free.restype = None
    L.agb_pattern_desc.argtypes = [C.c_void_p]
    L.agb_pattern_desc.restype = C.POINTER(Desc)
    L.agb_pattern_from_desc.argtypes = [C.POINTER(Desc), C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.agb_pattern_regex.argtypes = [C.c_void_p]
    L.agb_pattern_regex.restype = C.POINTER(Regex)
    L.agb_pattern_wide.argtypes = [C.c_void_p]
    L.agb_pattern_wide.restype = C.POINTER(Wide)
    L.agb_pattern_from_regex.argtypes = [C.POINTER(Desc), C.POINTER(Regex), C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.agb_scan_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(Result)]
    L.agb_scan_host.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(Result)]
    L.agb_scan_fd.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(Result)]
    L.agb_scan_host_windowed.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(Result)]
    L.agb_scan_fd_windowed.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(Result)]
    L.agb_scan_set.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.c_uint32, C.c_int, C.c_void_p, C.c_uint64,
                               C.POINTER(Result), C.POINTER(Result)]
    L.agb_bestmatch_device.argtypes = [C.c_char_p, C.POINTER(Options), C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                       C.POINTER(C.c_int), C.POINTER(Result), C.c_char_p, C.c_size_t]
    L.agb_corpus_fill_device.argtypes = [C.POINTER(CorpusSpec), C.c_void_p, C.c_void_p]
    L.agb_corpus_fill_host.argtypes = [C.POINTER(CorpusSpec), C.c_void_p]
    L.agb_fill_ordinals.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    L.agb_fill_ordinals.restype = None
    L.agb_text_from_host.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)]
    L.agb_text_from_fd.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    L.agb_text_free.argtypes = [C.c_void_p]
    L.agb_text_free.restype = None
    L.agb_text_size.argtypes = [C.c_void_p]
    L.agb_text_size.restype = C.c_uint64
    L.agb_text_device.argtypes = [C.c_void_p]
    L.agb_text_device.restype = C.c_void_p
    L.agb_scan_text.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_uint64, C.POINTER(Result)]
    L.agb_comm_unique_id.argtypes = [C.c_void_p]
    L.agb_comm_init.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p]
    L.agb_comm_free.argtypes = [C.c_void_p]
    L.agb_comm_free.restype = None
    L.agb_comm_world.argtypes = [C.c_void_p]
    L.agb_comm_rank.argtypes = [C.c_void_p]
    L.agb_shard_halo.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p]
    L.agb_scan_sharded.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p, C.c_uint64,
                                   C.c_void_p, C.POINTER(Result)]
    L.agb_scan_shard_local.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int,
                                       C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(Result), C.POINTER(ShardPart)]
    L.agb_bestmatch_sharded.argtypes = [C.c_char_p, C.POINTER(Options), C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p,
                                        C.c_uint64, C.c_void_p, C.POINTER(C.c_int), C.POINTER(Result), C.c_char_p, C.c_size_t]
    L.agb_last_error.restype = C.c_char_p
    L.agb_version.restype = C.c_char_p
    L.agb_kernel_launches.restype = C.c_uint64
    _lib = L
    return L
