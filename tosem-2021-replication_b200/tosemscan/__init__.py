"""tosemscan - Python host mirror of include/tosemscan.h (ctypes over the C ABI).

The reference package ships no operator/plugin interface (SURVEY.md section 8b); this module is the thin
host layer the parity tests and bench.py use: numpy arrays in, numpy arrays out, every call
forwarded to ``libtosemscan.so`` (hand-written sm_90a CUDA).  There is NO CPU fallback: a
missing library or a missing GPU raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TOSEMSCAN_LIB") or os.path.join(_HERE, "libtosemscan.so")   # env override: tuning variants

K = 128
ALIGN = 128
EXT = {"py": 1, "cc": 2, "cpp": 3, "java": 4, "c": 5, "h": 6}
SCAN_ASSERT_EVENTS = 1
SCAN_HEADER_EVENTS = 2
SCAN_REV_B = 8            # docs/SPEC.md section 4b (golden G1)
TSM_E_CAPACITY = -3

FILE_STAT = np.dtype([("n_lines", "<u4"), ("n_assert", "<u4"), ("n_headers", "<u4"),
                      ("n_fixture", "<u4"), ("digest", "<u8")])
ASSERT_EVENT = np.dtype([("file", "<u4"), ("line_off", "<u4"), ("stmt_off", "<u4"),
                         ("stmt_len", "<u2"), ("cat", "<u2"), ("ident_off", "<u4"),
                         ("ident_len", "<u2"), ("pad", "<u2"), ("stmt_hash", "<u8")])
HEADER_EVENT = np.dtype([("file", "<u4"), ("line_off", "<u4"), ("line_len", "<u4"), ("kind", "<u4")])
DIFF_DETAIL = np.dtype([("hunks_add", "<i8"), ("hunks_del", "<i8"), ("hunks_mod", "<i8"),
                        ("added_assert", "<i8"), ("removed_assert", "<i8")])
ORIGIN = np.dtype([("change", "<i4"), ("line", "<i4")])   # tsm_origin: the change that inserted a line, 1-based line there
CASE = np.dtype([("pair", "<i4"), ("line", "<i4"), ("n_lines", "<i4"), ("n_assert", "<i4"), ("n_changed", "<i4"),
                 ("n_changed_assert", "<i4"), ("match", "<i4")])   # tsm_case: one test case of one side of a revision pair
SMELL_TEST = np.dtype([("file", "<i4"), ("line", "<i4"), ("body_lines", "<i4"), ("n_assert", "<i4"), ("smells", "<u4"),
                       ("n_instances", "<i4")])   # tsm_smell_test: one test of the corpus (docs/SPEC.md section 18)
SMELLS = ["empty", "assertion_free", "duplicate_assert", "redundant_assert", "conditional_logic", "exception_handling", "sleepy",
          "print", "ignored"]                   # bit k of tsm_smell_test.smells and of line_smell is SMELLS[k]
LEX_TEST = np.dtype([("n_stmts", "<i4"), ("n_unexplained", "<i4"), ("n_magic", "<i4"), ("n_locals", "<i4"), ("smells", "<u4"),
                     ("n_instances", "<i4")])   # tsm_lex_test: the lexical smells of one test (docs/SPEC.md section 25)
LSMELLS = ["assertion_roulette", "magic_number", "suboptimal_assert", "mystery_guest",
           "obscure_setup"]                     # bit k of tsm_lex_test.smells and of line_lsmell is LSMELLS[k]
TEST_CHURN = np.dtype([("case_idx", "<i4"), ("instances", "<i4", (9,)), ("churned", "<i4", (9,))])   # tsm_test_churn (section 19)
LEX_CHURN = np.dtype([("instances", "<i4", (5,)), ("churned", "<i4", (5,))])   # tsm_lex_churn (section 26), smell k = LSMELLS[k]
MOVE_BLOCK = np.dtype([("line", "<i8"), ("partner", "<i8"), ("n_lines", "<i4"),
                       ("n_assert", "<i4")])   # tsm_move_block: one moved block of one side (docs/SPEC.md section 20)
SIMILAR_PAIR = np.dtype([("a", "<i4"), ("b", "<i4"), ("lcs", "<u4"),
                         ("score", "<u4")])   # tsm_similar_pair: two similar tests, a < b (docs/SPEC.md section 23)
SIMILAR_EVENT = np.dtype([("status", "<i4"), ("old_a", "<i4"), ("old_b", "<i4"), ("a", "<i4"), ("b", "<i4"), ("old_lcs", "<u4"),
                          ("old_score", "<u4"), ("lcs", "<u4"), ("score", "<u4")])   # tsm_similar_event (docs/SPEC.md section 24)
SIMILAR_STATUSES = ["changed", "removed", "dropped", "diverged", "created", "copied", "converged"]   # SIMILAR_EVENT status
LINK_TEST = np.dtype([("file", "<i4"), ("line", "<i4"), ("calls", "<i4"), ("linked_calls", "<i4"), ("links", "<i4"),
                      ("function_links", "<i4"), ("focal_links", "<i4"),
                      ("flags", "<u4")])   # tsm_link_test: one test of a test file and its links (docs/SPEC.md section 27)
LINK = np.dtype([("test", "<i4"), ("name_def", "<i4"), ("target", "<i4"), ("n_defs", "<i4"), ("calls", "<i4"), ("line", "<i4"),
                 ("byte", "<i4")])   # tsm_link: one (test, name) link, its target definition or -1 and its first call
LINK_DEF = np.dtype([("file", "<i4"), ("line", "<i4"), ("name_off", "<i4"), ("name_len", "<i4"), ("kind", "<i4"), ("tests", "<i4"),
                     ("tests_by_name", "<i4"), ("calls", "<i4")])   # tsm_link_def: one definition of a production file
LINK_EAGER, LINK_LAZY = 1, 2                     # bits of LINK_TEST flags
LINK_KINDS = {1: "function", 2: "class"}         # LINK_DEF kind
LINK_EVENT = np.dtype([("event", "<i4"), ("cause", "<i4"), ("old_test", "<i4"), ("test", "<i4"), ("old_link", "<i4"), ("link", "<i4"),
                       ("old_calls", "<i4"), ("calls", "<i4"), ("old_defs", "<i4"),
                       ("defs", "<i4")])   # tsm_link_event: one row of the link churn (docs/SPEC.md section 28), -1 where absent
LINK_EVENTS = ["added", "removed", "retargeted", "redefined", "eager_introduced", "eager_removed", "lazy_introduced",
               "lazy_removed"]                   # LINK_EVENT event
LINK_CAUSES = ["test", "call", "definition"]     # LINK_EVENT cause of added / removed (-1 for the others)
ASSERT_EDIT = np.dtype([("rev", "<i8"), ("aev", "<i8"), ("score", "<i4"), ("_pad", "<i4")])   # tsm_assert_edit: event indices

# every symbol include/tosemscan.h declares (tests check the library exports exactly these)
SYMBOLS = ["tsm_abi_version", "tsm_strerror", "tsm_category_name", "tsm_create", "tsm_destroy", "tsm_scan",
           "tsm_upload", "tsm_scan_resident", "tsm_download", "tsm_device_counts", "tsm_last_launch_count", "tsm_last_kernel_ms", "tsm_kernel_ms_stats",
           "tsm_diff_pairs", "tsm_diff_pairs_detail", "tsm_statements", "tsm_line_hashes", "tsm_diff_upload", "tsm_diff_resident", "tsm_diff_last_ms",
           "tsm_diff_pairs_asserts", "tsm_diff_resident_asserts", "tsm_reduce", "tsm_host_alloc", "tsm_host_free", "tsm_layout", "tsm_gen_sizes",
           "tsm_gen_fill", "tsm_gen_edit", "tsm_gen_pair_sizes", "tsm_gen_pair_fill", "tsm_similarity", "tsm_similarity_last_ms",
           "tsm_diff_pairs_marks", "tsm_blame_pairs", "tsm_blame_last_ms", "tsm_clones", "tsm_clones_last_ms",
           "tsm_diff_pairs_cases", "tsm_diff_pairs_assert_edits", "tsm_assert_edits_last_ms", "tsm_smells", "tsm_smells_last_ms",
           "tsm_diff_pairs_smells", "tsm_diff_smells_last_ms", "tsm_diff_pairs_moves", "tsm_moves_last_ms", "tsm_clones_blind",
           "tsm_clones_blind_last_ms", "tsm_clone_churn", "tsm_clone_churn_last_ms", "tsm_similar_tests", "tsm_similar_tests_last_ms",
           "tsm_similar_churn", "tsm_similar_churn_last_ms", "tsm_smells_lexical", "tsm_smells_lexical_last_ms",
           "tsm_diff_pairs_smells_lexical", "tsm_diff_smells_lexical_last_ms", "tsm_test_links", "tsm_test_links_last_ms",
           "tsm_focal_stems", "tsm_link_churn", "tsm_link_churn_last_ms"]
FRAG_STATES = ["kept", "edited", "whole"]          # tsm_clone_churn state[j] (docs/SPEC.md section 22)
CLONE_STATUSES = ["untouched", "changed", "removed", "diverged", "dropped", "created", "copied", "joined"]   # status[c]


class TsmError(RuntimeError):
    def __init__(self, status, what):
        self.status = status
        super().__init__(f"{what}: {lib().tsm_strerror(status).decode()} ({status})")


class _Corpus(C.Structure):
    _fields_ = [("arena", C.c_void_p), ("off", C.c_void_p), ("len", C.c_void_p), ("ext", C.c_void_p),
                ("grp", C.c_void_p), ("n_files", C.c_int32), ("n_groups", C.c_int32)]


class _Result(C.Structure):
    _fields_ = [("stats", C.c_void_p), ("group_counts", C.c_void_p), ("global_counts", C.c_void_p),
                ("aev", C.c_void_p), ("aev_cap", C.c_int64), ("n_aev", C.c_int64),
                ("hev", C.c_void_p), ("hev_cap", C.c_int64), ("n_hev", C.c_int64),
                ("totals", C.c_int64 * 4)]


class _LineMarks(C.Structure):
    _fields_ = [("line_base_old", C.c_void_p), ("line_base_new", C.c_void_p),
                ("dels", C.c_void_p), ("del_cap", C.c_int64), ("n_old", C.c_int64),
                ("ins", C.c_void_p), ("ins_cap", C.c_int64), ("n_new", C.c_int64)]


class _DiffAsserts(C.Structure):
    _fields_ = [("added_counts", C.c_void_p), ("removed_counts", C.c_void_p),
                ("aev", C.c_void_p), ("aev_cap", C.c_int64), ("n_aev", C.c_int64),
                ("rev", C.c_void_p), ("rev_cap", C.c_int64), ("n_rev", C.c_int64)]


class _DiffCases(C.Structure):
    _fields_ = [("old_cases", C.c_void_p), ("old_cap", C.c_int64), ("n_old", C.c_int64),
                ("new_cases", C.c_void_p), ("new_cap", C.c_int64), ("n_new", C.c_int64)]


class _DiffSmells(C.Structure):
    _fields_ = [("cases", _DiffCases),
                ("old_tests", C.c_void_p), ("old_churn", C.c_void_p), ("old_test_cap", C.c_int64), ("n_old_tests", C.c_int64),
                ("new_tests", C.c_void_p), ("new_churn", C.c_void_p), ("new_test_cap", C.c_int64), ("n_new_tests", C.c_int64)]


class _DiffLexSmells(C.Structure):
    _fields_ = [("old_lex", C.c_void_p), ("old_churn", C.c_void_p), ("new_lex", C.c_void_p), ("new_churn", C.c_void_p)]


class _DiffMoves(C.Structure):
    _fields_ = [("marks", _LineMarks),
                ("old_blocks", C.c_void_p), ("old_cap", C.c_int64), ("n_old_blocks", C.c_int64),
                ("new_blocks", C.c_void_p), ("new_cap", C.c_int64), ("n_new_blocks", C.c_int64)]


class _CloneResult(C.Structure):
    _fields_ = [("line_base", C.c_void_p), ("file_dup", C.c_void_p), ("file_dup_assert", C.c_void_p),
                ("class_base", C.c_void_p), ("class_len", C.c_void_p), ("class_cap", C.c_int64), ("n_classes", C.c_int64),
                ("member", C.c_void_p), ("member_cap", C.c_int64), ("n_members", C.c_int64)]


class _BlindResult(C.Structure):
    _fields_ = [("kept_base", C.c_void_p), ("kept_line", C.c_void_p), ("blind_hash", C.c_void_p), ("file_kept_assert", C.c_void_p),
                ("kept_cap", C.c_int64), ("n_kept", C.c_int64)]


class _SimilarResult(C.Structure):
    _fields_ = [("tests", C.c_void_p), ("test_kept", C.c_void_p), ("test_cap", C.c_int64), ("n_tests", C.c_int64),
                ("pairs", C.c_void_p), ("pair_cap", C.c_int64), ("n_pairs", C.c_int64),
                ("class_base", C.c_void_p), ("class_cap", C.c_int64), ("n_classes", C.c_int64),
                ("member", C.c_void_p), ("member_cap", C.c_int64), ("n_members", C.c_int64), ("n_candidates", C.c_int64)]


class _LinksResult(C.Structure):
    _fields_ = [("tests", C.c_void_p), ("test_cap", C.c_int64), ("n_tests", C.c_int64), ("links", C.c_void_p), ("link_cap", C.c_int64),
                ("n_links", C.c_int64), ("defs", C.c_void_p), ("def_cap", C.c_int64), ("n_defs", C.c_int64)]


class _LinkChurnSide(C.Structure):
    _fields_ = [("links", _LinksResult), ("match", C.c_void_p), ("change", C.c_void_p)]


class _SimilarChurnSide(C.Structure):
    _fields_ = [("tests", C.c_void_p), ("test_kept", C.c_void_p), ("match", C.c_void_p), ("change", C.c_void_p), ("test_cap", C.c_int64),
                ("n_tests", C.c_int64), ("n_candidates", C.c_int64)]


class _CloneChurnSide(C.Structure):
    _fields_ = [("clones", _CloneResult), ("blind", _BlindResult), ("changed", C.c_void_p), ("changed_assert", C.c_void_p),
                ("state", C.c_void_p), ("class_counts", C.c_void_p), ("status", C.c_void_p)]


_lib = None


def lib():
    """Load libtosemscan.so (built in-tree by __graft_entry__.build() / make). Fails loudly."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(f"{LIB_PATH} is missing: build it with `make -C tosem-2021-replication_b200` "
                              "(there is no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        L.tsm_abi_version.restype = C.c_int
        L.tsm_strerror.restype = C.c_char_p
        L.tsm_strerror.argtypes = [C.c_int]
        L.tsm_category_name.restype = C.c_char_p
        L.tsm_category_name.argtypes = [C.c_int]
        L.tsm_create.restype = C.c_int
        L.tsm_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int64, C.c_int32, C.c_int32, C.c_int64]
        L.tsm_destroy.restype = None
        L.tsm_destroy.argtypes = [C.c_void_p]
        L.tsm_scan.restype = C.c_int
        L.tsm_scan.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Result), C.c_uint32, C.c_void_p]
        L.tsm_upload.restype = C.c_int
        L.tsm_upload.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_void_p]
        L.tsm_scan_resident.restype = C.c_int
        L.tsm_scan_resident.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        L.tsm_download.restype = C.c_int
        L.tsm_download.argtypes = [C.c_void_p, C.POINTER(_Result), C.c_void_p]
        L.tsm_device_counts.restype = C.c_int
        L.tsm_device_counts.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64)]
        L.tsm_last_launch_count.restype = C.c_int
        L.tsm_last_launch_count.argtypes = [C.c_void_p]
        L.tsm_last_kernel_ms.restype = C.c_int
        L.tsm_last_kernel_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_kernel_ms_stats.restype = C.c_int
        L.tsm_kernel_ms_stats.argtypes = [C.c_void_p, C.POINTER(C.c_double * 4), C.POINTER(C.c_int64), C.c_int]
        L.tsm_diff_pairs.restype = C.c_int
        L.tsm_diff_pairs.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsm_diff_pairs_detail.restype = C.c_int
        L.tsm_diff_pairs_detail.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.c_void_p]
        L.tsm_statements.restype = C.c_int
        L.tsm_statements.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                     C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_line_hashes.restype = C.c_int
        L.tsm_line_hashes.argtypes = [C.c_void_p, C.POINTER(_Corpus)] + [C.c_void_p] * 4 + [C.c_int64, C.POINTER(C.c_int64), C.c_int32,
                                      C.c_void_p, C.c_void_p]
        L.tsm_reduce.restype = C.c_int
        L.tsm_reduce.argtypes = [C.c_void_p] * 4 + [C.c_int32] * 4 + [C.c_void_p] * 3
        L.tsm_host_alloc.restype = C.c_void_p
        L.tsm_host_alloc.argtypes = [C.c_int64]
        L.tsm_host_free.restype = None
        L.tsm_host_free.argtypes = [C.c_void_p]
        L.tsm_layout.restype = C.c_int64
        L.tsm_layout.argtypes = [C.c_void_p, C.c_int32, C.c_void_p]
        L.tsm_gen_sizes.restype = C.c_int
        L.tsm_gen_sizes.argtypes = [C.c_uint64, C.c_int32, C.c_int, C.c_int32, C.c_int32, C.c_int32,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]
        L.tsm_gen_fill.restype = C.c_int
        L.tsm_gen_fill.argtypes = [C.c_uint64, C.c_int32, C.c_int, C.c_int32, C.c_int32,
                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsm_gen_edit.restype = C.c_int64
        L.tsm_gen_edit.argtypes = [C.c_uint64, C.c_void_p, C.c_int32, C.c_double, C.c_void_p, C.c_int64]
        L.tsm_gen_pair_sizes.restype = C.c_int
        L.tsm_gen_pair_sizes.argtypes = [C.c_uint64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double,
                                         C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsm_gen_pair_fill.restype = C.c_int
        L.tsm_gen_pair_fill.argtypes = [C.c_uint64, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double] + [C.c_void_p] * 7
        L.tsm_diff_upload.restype = C.c_int
        L.tsm_diff_upload.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p]
        L.tsm_diff_resident.restype = C.c_int
        L.tsm_diff_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.tsm_diff_pairs_asserts.restype = C.c_int
        L.tsm_diff_pairs_asserts.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_DiffAsserts), C.c_void_p]
        L.tsm_diff_resident_asserts.restype = C.c_int
        L.tsm_diff_resident_asserts.argtypes = [C.c_void_p] * 4 + [C.POINTER(_DiffAsserts), C.c_void_p]
        L.tsm_diff_last_ms.restype = C.c_int
        L.tsm_diff_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 3)]
        L.tsm_similarity.restype = C.c_int
        L.tsm_similarity.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_int64,
                                     C.c_void_p, C.c_void_p]
        L.tsm_similarity_last_ms.restype = C.c_int
        L.tsm_similarity_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 3)]
        L.tsm_diff_pairs_marks.restype = C.c_int
        L.tsm_diff_pairs_marks.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_LineMarks), C.c_void_p]
        L.tsm_diff_pairs_cases.restype = C.c_int
        L.tsm_diff_pairs_cases.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_DiffCases), C.c_void_p]
        L.tsm_diff_pairs_assert_edits.restype = C.c_int
        L.tsm_diff_pairs_assert_edits.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_DiffAsserts), C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_blame_pairs.restype = C.c_int
        L.tsm_blame_pairs.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 10 + \
            [C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_blame_last_ms.restype = C.c_int
        L.tsm_blame_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
        L.tsm_clones.restype = C.c_int
        L.tsm_clones.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_int32, C.POINTER(_CloneResult), C.c_void_p]
        L.tsm_clones_last_ms.restype = C.c_int
        L.tsm_clones_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 3)]
        L.tsm_clones_blind.restype = C.c_int
        L.tsm_clones_blind.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_int32, C.POINTER(_BlindResult), C.POINTER(_CloneResult),
                                       C.c_void_p]
        L.tsm_clones_blind_last_ms.restype = C.c_int
        L.tsm_clones_blind_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_smells.restype = C.c_int
        L.tsm_smells.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64),
                                 C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_smells_last_ms.restype = C.c_int
        L.tsm_smells_lexical.restype = C.c_int
        L.tsm_smells_lexical.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64,
                                         C.POINTER(C.c_int64), C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_smells_lexical_last_ms.restype = C.c_int
        L.tsm_smells_lexical_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_test_links.restype = C.c_int
        L.tsm_test_links.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.POINTER(_LinksResult), C.c_void_p]
        L.tsm_test_links_last_ms.restype = C.c_int
        L.tsm_test_links_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_link_churn.restype = C.c_int
        L.tsm_link_churn.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_void_p, C.c_void_p, C.c_int64, C.POINTER(_LinkChurnSide), C.POINTER(_LinkChurnSide), C.c_void_p,
                                     C.c_int64, C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_link_churn_last_ms.restype = C.c_int
        L.tsm_link_churn_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_focal_stems.restype = C.c_int
        L.tsm_focal_stems.argtypes = [C.POINTER(C.c_char_p), C.c_void_p, C.c_int32, C.c_void_p]
        L.tsm_similar_tests.restype = C.c_int
        L.tsm_similar_tests.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.c_int32, C.c_int32, C.POINTER(_SimilarResult), C.c_void_p]
        L.tsm_similar_tests_last_ms.restype = C.c_int
        L.tsm_similar_tests_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_similar_churn.restype = C.c_int
        L.tsm_similar_churn.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                        C.c_int32, C.POINTER(_SimilarChurnSide), C.POINTER(_SimilarChurnSide), C.c_void_p, C.c_int64,
                                        C.POINTER(C.c_int64), C.c_void_p]
        L.tsm_similar_churn_last_ms.restype = C.c_int
        L.tsm_similar_churn_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_smells_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_diff_pairs_smells.restype = C.c_int
        L.tsm_diff_pairs_smells.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_DiffSmells), C.c_void_p]
        L.tsm_diff_smells_last_ms.restype = C.c_int
        L.tsm_diff_smells_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_diff_pairs_smells_lexical.restype = C.c_int
        L.tsm_diff_pairs_smells_lexical.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_DiffSmells), C.POINTER(_DiffLexSmells), C.c_void_p]
        L.tsm_diff_smells_lexical_last_ms.restype = C.c_int
        L.tsm_diff_smells_lexical_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_diff_pairs_moves.restype = C.c_int
        L.tsm_diff_pairs_moves.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus)] + [C.c_void_p] * 3 + \
            [C.POINTER(_DiffMoves), C.c_void_p]
        L.tsm_moves_last_ms.restype = C.c_int
        L.tsm_moves_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        L.tsm_clone_churn.restype = C.c_int
        L.tsm_clone_churn.argtypes = [C.c_void_p, C.POINTER(_Corpus), C.POINTER(_Corpus), C.c_void_p, C.c_void_p, C.c_int64, C.c_int32,
                                      C.c_int32, C.POINTER(_CloneChurnSide), C.POINTER(_CloneChurnSide), C.c_void_p]
        L.tsm_clone_churn_last_ms.restype = C.c_int
        L.tsm_clone_churn_last_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float * 4)]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def focal_stems(paths, role):
    """The naming convention of docs/SPEC.md section 27 (tsm_focal_stems): per path, the id of a production file's base name
    without its extension, or of a test file's focal stem (-1 when it is empty).  paths: str or bytes; role: nonzero = test file."""
    n = len(paths)
    arr = (C.c_char_p * max(n, 1))(*[p.encode() if isinstance(p, str) else bytes(p) for p in paths])
    role = np.ascontiguousarray(role, np.uint8)
    stem = np.zeros(max(n, 1), np.int32)
    rc = lib().tsm_focal_stems(arr, _p(role), n, _p(stem))
    if rc:
        raise TsmError(rc, "tsm_focal_stems")
    return stem[:n]


def category_name(i):
    return lib().tsm_category_name(i).decode()


class _Pinned:
    """A pinned host allocation (cudaHostAlloc) exposed as a numpy uint8 array."""

    def __init__(self, nbytes):
        self.ptr = lib().tsm_host_alloc(nbytes)
        self.nbytes = nbytes
        if not self.ptr:
            raise MemoryError("tsm_host_alloc failed")
        self.array = np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(self.ptr))

    def __del__(self):
        if getattr(self, "ptr", None):
            lib().tsm_host_free(self.ptr)
            self.ptr = None


def host_buffer(nbytes, pinned=True):
    """uint8 buffer for an arena: pinned when a GPU is present and pinned=True, else plain numpy."""
    if pinned:
        try:
            pin = _Pinned(max(int(nbytes), ALIGN))
            arr = pin.array
            arr[:] = 0
            return arr, pin
        except MemoryError:
            pass
    return np.zeros(max(int(nbytes), ALIGN), np.uint8), None


class Corpus:
    """Packed corpus of docs/SPEC.md section 1 (arena + int32 offset index + per-file tags)."""

    def __init__(self, arena, off, length, ext, grp=None, n_groups=1, keep=None):
        self.arena = arena
        self.off = np.ascontiguousarray(off, np.int32)
        self.len = np.ascontiguousarray(length, np.int32)
        self.ext = np.ascontiguousarray(ext, np.uint8)
        self.grp = np.zeros(len(self.len), np.uint16) if grp is None else np.ascontiguousarray(grp, np.uint16)
        self.n_groups = int(n_groups)
        self._keep = keep
        if keep is not None:                                 # pinned arena: pin the index too (tsm_scan copies it every call;
            self._pin_index()                               # from pageable memory those copies are staged and block the host)

    def _pin_index(self):
        pins = []
        for name in ("off", "len", "ext", "grp"):
            a = getattr(self, name)
            try:
                pin = _Pinned(max(a.nbytes, ALIGN))
            except MemoryError:
                return
            b = pin.array[:a.nbytes].view(a.dtype)
            b[:] = a
            setattr(self, name, b)
            pins.append(pin)
        self._index_pins = pins

    @property
    def n_files(self):
        return len(self.len)

    @property
    def source_bytes(self):
        return int(self.len.astype(np.int64).sum())

    @property
    def algorithmic_bytes(self):
        """SURVEY.md section 8d: every source byte once + the int32 offset index."""
        return self.source_bytes + 4 * (self.n_files + 1)

    def c_struct(self):
        return _Corpus(_p(self.arena), _p(self.off), _p(self.len), _p(self.ext), _p(self.grp),
                       self.n_files, self.n_groups)

    def file_bytes(self, i):
        o = int(self.off[i])
        return self.arena[o:o + int(self.len[i])].tobytes()


def pack(files, exts, grps=None, n_groups=1, pinned=False):
    """Pack bytes objects end to end with 128-B aligned starts."""
    n = len(files)
    length = np.array([len(f) for f in files], np.int32)
    off = np.zeros(n + 1, np.int32)
    total = lib().tsm_layout(_p(length), n, _p(off))
    if total < 0:
        raise ValueError("corpus does not fit an int32-indexed arena (2 GiB): pack it in batches")
    arena, keep = host_buffer(total, pinned)
    for i, f in enumerate(files):
        if f:
            arena[off[i]:off[i] + len(f)] = np.frombuffer(f, np.uint8)
    return Corpus(arena, off, length, exts, grps, n_groups, keep)


def gen_corpus(seed, n_files, size_law=0, fixed_size=4096, first_index=0, index_stride=1, n_groups=1,
               pinned=True, threads=None):
    """Synthetic corpus of SURVEY.md section 8d (deterministic, std::mt19937_64 in the C++ host library)."""
    L = lib()
    length = np.zeros(n_files, np.int32)
    ext = np.zeros(n_files, np.uint8)
    grp = np.zeros(n_files, np.uint16)
    rc = L.tsm_gen_sizes(seed, n_files, size_law, fixed_size, first_index, index_stride, _p(length), _p(ext),
                         _p(grp), n_groups)
    if rc:
        raise TsmError(rc, "tsm_gen_sizes")
    off = np.zeros(n_files + 1, np.int32)
    total = L.tsm_layout(_p(length), n_files, _p(off))
    if total < 0:
        raise ValueError("corpus does not fit an int32-indexed arena")
    arena, keep = host_buffer(total, pinned)
    # files are independent: fill slices on all host cores (ctypes releases the GIL)
    nthr = max(1, min(threads or (os.cpu_count() or 1), 64, (n_files + 255) // 256))
    bounds = [n_files * t // nthr for t in range(nthr + 1)]

    def fill(t):
        a, b = bounds[t], bounds[t + 1]
        if a == b:
            return 0
        return L.tsm_gen_fill(seed, b - a, size_law, first_index + a * index_stride, index_stride,
                              _p(off[a:b + 1]), _p(length[a:b]), _p(ext[a:b]), _p(arena))
    if nthr == 1:
        rcs = [fill(0)]
    else:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(nthr) as ex:
            rcs = list(ex.map(fill, range(nthr)))
    if any(rcs):
        raise TsmError([r for r in rcs if r][0], "tsm_gen_fill")
    return Corpus(arena, off, length, ext, grp, n_groups, keep)


def gen_pair_sizes(seed, n_pairs, cap=65536, lam=6.0, index=None, first_index=0, index_stride=1, threads=None):
    """(len_old, len_new, ext) of the logical pairs index[...] (or first_index + i*stride) of BASELINE config C5."""
    L = lib()
    idx = None if index is None else np.ascontiguousarray(index, np.int32)
    n = n_pairs if idx is None else len(idx)
    lo, ln, ext = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint8)
    nthr = max(1, min(threads or (os.cpu_count() or 1), 64, (n + 255) // 256))
    bounds = [n * t // nthr for t in range(nthr + 1)]

    def sizes(t):
        a, b = bounds[t], bounds[t + 1]
        if a == b:
            return 0
        return L.tsm_gen_pair_sizes(seed, b - a, None if idx is None else _p(idx[a:b]), first_index + a * index_stride, index_stride,
                                    cap, float(lam), _p(lo[a:b]), _p(ln[a:b]), _p(ext[a:b]))
    _run_threads(sizes, nthr, "tsm_gen_pair_sizes")
    return lo, ln, ext


def _run_threads(fn, nthr, what):
    if nthr == 1:
        rcs = [fn(0)]
    else:
        from concurrent.futures import ThreadPoolExecutor
        with ThreadPoolExecutor(nthr) as ex:
            rcs = list(ex.map(fn, range(nthr)))
    if any(rcs):
        raise TsmError([r for r in rcs if r][0], what)


def gen_pairs(seed, n_pairs, cap=65536, lam=6.0, first_index=0, index_stride=1, pinned=True, threads=None, index=None, sizes=None):
    """BASELINE config C5: (olds, news) corpora of revision pairs (SURVEY.md section 8d), generated in C++.  `index` picks
    logical pairs by number (a rank's share of a size-balanced deal); `sizes` = gen_pair_sizes of the same pairs, if known."""
    L = lib()
    idx = None if index is None else np.ascontiguousarray(index, np.int32)
    n = n_pairs if idx is None else len(idx)
    lo, ln, ext = sizes if sizes is not None else gen_pair_sizes(seed, n, cap, lam, idx, first_index, index_stride, threads)
    oo, on = np.zeros(n + 1, np.int32), np.zeros(n + 1, np.int32)
    to, tn = L.tsm_layout(_p(lo), n, _p(oo)), L.tsm_layout(_p(ln), n, _p(on))
    if to < 0 or tn < 0:
        raise ValueError("pairs do not fit an int32-indexed arena")
    ao, ko = host_buffer(to, pinned)
    an, kn = host_buffer(tn, pinned)
    nthr = max(1, min(threads or (os.cpu_count() or 1), 64, (n + 255) // 256))
    bounds = [n * t // nthr for t in range(nthr + 1)]

    def fill(t):
        a, b = bounds[t], bounds[t + 1]
        if a == b:
            return 0
        return L.tsm_gen_pair_fill(seed, b - a, None if idx is None else _p(idx[a:b]), first_index + a * index_stride, index_stride,
                                   cap, float(lam), _p(ext[a:b]), _p(oo[a:b + 1]), _p(lo[a:b]), _p(ao), _p(on[a:b + 1]), _p(ln[a:b]), _p(an))
    _run_threads(fill, nthr, "tsm_gen_pair_fill")
    return Corpus(ao, oo, lo, ext, None, 1, ko), Corpus(an, on, ln, ext.copy(), None, 1, kn)


def gen_edit(seed, src: bytes, lam=6.0) -> bytes:
    buf = np.frombuffer(src, np.uint8) if src else np.zeros(1, np.uint8)
    out = np.zeros(len(src) + 64 * 256 * int(lam * 4 + 16), np.uint8)
    n = lib().tsm_gen_edit(seed, _p(buf), len(src), float(lam), _p(out), out.size)
    if n < 0:
        raise ValueError("tsm_gen_edit failed")
    return out[:n].tobytes()


class Scanner:
    """One CUDA device context (tsm_ctx)."""

    def __init__(self, device=0, max_arena_bytes=1 << 26, max_files=1 << 16, max_groups=16, max_events=0):
        self._ctx = C.c_void_p()
        rc = lib().tsm_create(C.byref(self._ctx), device, max_arena_bytes, max_files, max_groups, max_events)
        if rc:
            raise TsmError(rc, "tsm_create")
        self.max_events = max_events if max_events else max_arena_bytes // 32 + max_files
        self._corpus = None

    def close(self):
        if self._ctx:
            lib().tsm_destroy(self._ctx)
            self._ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _result(self, n_files, n_groups, flags, event_cap, reuse=False):
        if reuse:                                            # pinned buffers kept by the Scanner: D2H at the link rate, no
            key = (n_files, n_groups)                        # allocation per call; the arrays are valid until the next such call
            if getattr(self, "_res_key", None) != key:
                bufs = [host_buffer(max(n_files, 1) * FILE_STAT.itemsize), host_buffer(n_groups * K * 8), host_buffer(K * 8)]
                self._res_pins = [b[1] for b in bufs]
                self._res_bufs = (bufs[0][0][:n_files * FILE_STAT.itemsize].view(FILE_STAT),
                                  bufs[1][0][:n_groups * K * 8].view(np.int64).reshape(n_groups, K), bufs[2][0][:K * 8].view(np.int64))
                self._res_key = key
            res = {"stats": self._res_bufs[0], "group_counts": self._res_bufs[1], "global_counts": self._res_bufs[2]}
        else:
            res = {"stats": np.zeros(n_files, FILE_STAT), "group_counts": np.zeros((n_groups, K), np.int64),
                   "global_counts": np.zeros(K, np.int64)}
        r = _Result(_p(res["stats"]), _p(res["group_counts"]), _p(res["global_counts"]), None, 0, 0, None, 0, 0)
        if flags & SCAN_ASSERT_EVENTS:
            res["assert_events"] = np.zeros(max(event_cap, 1), ASSERT_EVENT)
            r.aev, r.aev_cap = _p(res["assert_events"]), event_cap
        if flags & SCAN_HEADER_EVENTS:
            res["header_events"] = np.zeros(max(event_cap, 1), HEADER_EVENT)
            r.hev, r.hev_cap = _p(res["header_events"]), event_cap
        return res, r

    @staticmethod
    def _events_too_small(r, flags):
        """tsm_download's TSM_E_CAPACITY for host event arrays shorter than the scan's events (it reports both counts)."""
        return bool((flags & SCAN_ASSERT_EVENTS and r.n_aev > r.aev_cap) or (flags & SCAN_HEADER_EVENTS and r.n_hev > r.hev_cap))

    @staticmethod
    def _finish(res, r, flags):
        res["totals"] = np.array(list(r.totals), np.int64)
        if flags & SCAN_ASSERT_EVENTS:
            res["assert_events"] = res["assert_events"][:r.n_aev]
        if flags & SCAN_HEADER_EVENTS:
            res["header_events"] = res["header_events"][:r.n_hev]
        return res

    def scan(self, corpus, flags=0, stream=None, event_cap=None, reuse=False):
        """End-to-end host path: H2D + kernels + D2H (tsm_scan).  reuse=True: the per-file records and count tables land in
        pinned buffers the Scanner keeps (valid until the next scan with reuse=True)."""
        want_ev = flags & (SCAN_ASSERT_EVENTS | SCAN_HEADER_EVENTS)
        cap = int(event_cap if event_cap is not None else (max(corpus.source_bytes // 8 + 16, 1024) if want_ev else 0))
        res, r = self._result(corpus.n_files, corpus.n_groups, flags, cap, reuse)
        cs = corpus.c_struct()
        rc = lib().tsm_scan(self._ctx, C.byref(cs), C.byref(r), flags, stream)
        if rc == TSM_E_CAPACITY and self._events_too_small(r, flags):   # more events than `cap`: fetch them again, sized
            res, r = self._result(corpus.n_files, corpus.n_groups, flags, max(r.n_aev, r.n_hev), reuse)
            rc = lib().tsm_download(self._ctx, C.byref(r), stream)
        if rc:
            raise TsmError(rc, "tsm_scan")
        self._corpus = corpus                               # tsm_scan leaves this corpus resident: download() reads its results
        return self._finish(res, r, flags)

    def upload(self, corpus, stream=None):
        cs = corpus.c_struct()
        rc = lib().tsm_upload(self._ctx, C.byref(cs), stream)
        if rc:
            raise TsmError(rc, "tsm_upload")
        self._corpus = corpus

    def scan_resident(self, flags=0, stream=None):
        rc = lib().tsm_scan_resident(self._ctx, flags, stream)
        if rc:
            raise TsmError(rc, "tsm_scan_resident")

    def download(self, flags=0, stream=None, event_cap=None):
        c = self._corpus
        cap = int(event_cap if event_cap is not None else max(c.source_bytes // 8 + 16, 1024))
        res, r = self._result(c.n_files, c.n_groups, flags, cap)
        rc = lib().tsm_download(self._ctx, C.byref(r), stream)
        if rc == TSM_E_CAPACITY and self._events_too_small(r, flags):
            res, r = self._result(c.n_files, c.n_groups, flags, max(r.n_aev, r.n_hev))
            rc = lib().tsm_download(self._ctx, C.byref(r), stream)
        if rc:
            raise TsmError(rc, "tsm_download")
        return self._finish(res, r, flags)

    def device_counts(self):
        """(device pointer, n_int64) of the [n_groups+1][K]+4 count table, for the one allreduce."""
        ptr, n = C.c_void_p(), C.c_int64()
        rc = lib().tsm_device_counts(self._ctx, C.byref(ptr), C.byref(n))
        if rc:
            raise TsmError(rc, "tsm_device_counts")
        return ptr.value, n.value

    def last_launch_count(self):
        return lib().tsm_last_launch_count(self._ctx)

    def last_kernel_ms(self):
        """Device time of k_plan, k_scan, k_classify of the last scan (4th slot is 0: k_totals is fused)."""
        ms = (C.c_float * 4)()
        rc = lib().tsm_last_kernel_ms(self._ctx, C.byref(ms))
        if rc:
            raise TsmError(rc, "tsm_last_kernel_ms")
        return [float(x) for x in ms]

    def kernel_ms_stats(self, reset=False):
        """(sum of ms per kernel [plan, scan, classify, totals], number of scans) since the last reset."""
        sums, n = (C.c_double * 4)(), C.c_int64()
        rc = lib().tsm_kernel_ms_stats(self._ctx, C.byref(sums), C.byref(n), int(reset))
        if rc:
            raise TsmError(rc, "tsm_kernel_ms_stats")
        return [float(x) for x in sums], int(n.value)

    def line_hashes(self, corpus, ngram=0, stream=None):
        """S9: (line_base[n+1], line_hash, line_end, line_flag[, ngram_hash]) of every line, files in order."""
        cs = corpus.c_struct()
        base = np.zeros(corpus.n_files + 1, np.int64)
        n = C.c_int64()
        rc = lib().tsm_line_hashes(self._ctx, C.byref(cs), _p(base), None, None, None, 0, C.byref(n), 0, None, stream)
        if rc not in (0, -3):
            raise TsmError(rc, "tsm_line_hashes")
        t = max(int(n.value), 1)
        lh, le, lf = np.zeros(t, np.uint64), np.zeros(t, np.uint32), np.zeros(t, np.uint8)
        ng = np.zeros(t, np.uint64) if ngram else None
        if n.value:
            rc = lib().tsm_line_hashes(self._ctx, C.byref(cs), _p(base), _p(lh), _p(le), _p(lf), t, C.byref(n), int(ngram), _p(ng), stream)
            if rc:
                raise TsmError(rc, "tsm_line_hashes")
        m = int(n.value)
        out = (base, lh[:m], le[:m], lf[:m])
        return out + (ng[:m],) if ngram else out

    def reduce(self, flags, repo, case_id, n_repos, n_cases, stream=None):
        flags = np.ascontiguousarray(flags, np.uint8)
        repo = np.ascontiguousarray(repo, np.int32)
        case_id = np.ascontiguousarray(case_id, np.int32)
        n_rows, n_flags = flags.shape
        out = np.zeros((n_flags, n_repos), np.int64)
        cpr = np.zeros(n_repos, np.int64)
        rc = lib().tsm_reduce(self._ctx, _p(flags), _p(repo), _p(case_id), n_rows, n_flags, n_repos, n_cases,
                              _p(out), _p(cpr), stream)
        if rc:
            raise TsmError(rc, "tsm_reduce")
        return out, cpr

    def statements(self, corpus, stream=None):
        """SPEC section 10: (line_base[n+1], line_end[lines], line_kind[lines]); kind 0 blank, 1 statement start, 2 continuation."""
        cs = corpus.c_struct()
        base = np.zeros(corpus.n_files + 1, np.int64)
        n = C.c_int64()
        rc = lib().tsm_statements(self._ctx, C.byref(cs), _p(base), None, None, 0, C.byref(n), stream)
        if rc not in (0, -3):
            raise TsmError(rc, "tsm_statements")
        end = np.zeros(max(n.value, 1), np.uint32)
        kind = np.zeros(max(n.value, 1), np.uint8)
        rc = lib().tsm_statements(self._ctx, C.byref(cs), _p(base), _p(end), _p(kind), n.value, C.byref(n), stream)
        if rc:
            raise TsmError(rc, "tsm_statements")
        return base, end[:n.value], kind[:n.value]

    def diff_pairs(self, olds, news, stream=None, detail=False, asserts=False):
        """S8 churn per pair; with detail=True also the hunks of the canonical edit script (SPEC section 8).  asserts=True:
        (added, removed, detail, added_counts, removed_counts, added_events, removed_events) - the changed assertion lines,
        as [n_groups][K] tables by the side's group and as events (inserted lines of `news`, deleted lines of `olds`)."""
        n = olds.n_files
        added = np.zeros(n, np.int64)
        removed = np.zeros(n, np.int64)
        a, b = olds.c_struct(), news.c_struct()
        if asserts:
            det = np.zeros(max(n, 1), DIFF_DETAIL)
            cap = (olds.source_bytes + news.source_bytes) // 1024 + 4096   # a guess: more events cost one more call
            return (added, removed, det[:n]) + self._diff_asserts(
                lambda r: lib().tsm_diff_pairs_asserts(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(r),
                                                       stream), olds.n_groups, cap, "tsm_diff_pairs_asserts")
        if not detail:
            rc = lib().tsm_diff_pairs(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), stream)
            if rc:
                raise TsmError(rc, "tsm_diff_pairs")
            return added, removed
        det = np.zeros(max(n, 1), DIFF_DETAIL)
        rc = lib().tsm_diff_pairs_detail(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), stream)
        if rc:
            raise TsmError(rc, "tsm_diff_pairs_detail")
        return added, removed, det[:n]

    @staticmethod
    def _diff_asserts(call, n_groups, cap, what, events=None):
        """(added_counts, removed_counts, added_events, removed_events) of one tsm_diff_*_asserts call; arrays too small for
        the events (TSM_E_CAPACITY with both counts) are sized from the counts and the call is made again.  events(cap):
        the two event arrays of at least cap entries (default: new arrays)."""
        events = events or (lambda c: (np.zeros(max(c, 1), ASSERT_EVENT), np.zeros(max(c, 1), ASSERT_EVENT)))
        for _ in range(2):
            ac, rc_ = np.zeros((n_groups, K), np.int64), np.zeros((n_groups, K), np.int64)
            aev, rev = events(cap)
            r = _DiffAsserts(_p(ac), _p(rc_), _p(aev), cap, 0, _p(rev), cap, 0)
            rc = call(r)
            if rc == TSM_E_CAPACITY and max(r.n_aev, r.n_rev) > cap:
                cap = int(max(r.n_aev, r.n_rev))
                continue
            if rc:
                raise TsmError(rc, what)
            return ac, rc_, aev[:r.n_aev], rev[:r.n_rev]
        raise TsmError(TSM_E_CAPACITY, what)

    def diff_upload(self, olds, news, stream=None):
        """Both sides of the pairs to HBM, kept by the ctx (tsm_diff_upload)."""
        a, b = olds.c_struct(), news.c_struct()
        rc = lib().tsm_diff_upload(self._ctx, C.byref(a), C.byref(b), stream)
        if rc:
            raise TsmError(rc, "tsm_diff_upload")
        self._pairs = olds.n_files
        self._pair_groups = olds.n_groups
        self._pair_bytes = olds.source_bytes + news.source_bytes
        n = max(self._pairs, 1)                              # results land in pinned memory: D2H at the PCIe rate, no staging copy
        bufs = [host_buffer(n * 8), host_buffer(n * 8), host_buffer(n * DIFF_DETAIL.itemsize)]
        self._diff_pins = [b[1] for b in bufs]
        self._diff_out = (bufs[0][0][:self._pairs * 8].view(np.int64), bufs[1][0][:self._pairs * 8].view(np.int64),
                          bufs[2][0][:n * DIFF_DETAIL.itemsize].view(DIFF_DETAIL))

    def diff_resident(self, detail=True, stream=None, asserts=False, event_cap=None):
        """The diff kernels over the resident sides; returns (added, removed[, detail]) - buffers reused across calls.
        asserts=True: (added, removed, detail, added_counts, removed_counts, added_events, removed_events) as diff_pairs; the
        event arrays are pinned buffers kept by the Scanner too (valid until the next such call)."""
        added, removed, det = self._diff_out
        if asserts:
            cap = int(event_cap if event_cap is not None else self._pair_bytes // 1024 + 4096)
            return (added, removed, det[:self._pairs]) + self._diff_asserts(
                lambda r: lib().tsm_diff_resident_asserts(self._ctx, _p(added), _p(removed), _p(det), C.byref(r), stream),
                self._pair_groups, cap, "tsm_diff_resident_asserts", self._event_buffers)
        rc = lib().tsm_diff_resident(self._ctx, _p(added), _p(removed), _p(det) if detail else None, stream)
        if rc:
            raise TsmError(rc, "tsm_diff_resident")
        return (added, removed, det[:self._pairs]) if detail else (added, removed)

    def _event_buffers(self, cap):
        """Two pinned event arrays of at least cap entries, grown when a call needs more (a fresh pageable array per call
        costs more host time than the classification of a C5 batch)."""
        if getattr(self, "_ev_cap", 0) < cap:
            bufs = [host_buffer(cap * ASSERT_EVENT.itemsize) for _ in range(2)]
            self._ev_pins = [b[1] for b in bufs]
            self._ev_bufs = tuple(b[0][:cap * ASSERT_EVENT.itemsize].view(ASSERT_EVENT) for b in bufs)
            self._ev_cap = cap
        return self._ev_bufs

    def diff_last_ms(self):
        """Device time of the last diff call: [k_scan over both sides, k_diff_small, k_myers + k_myers_trace of the pairs it left over] in ms."""
        ms = (C.c_float * 3)()
        lib().tsm_diff_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def diff_marks(self, olds, news, stream=None, cap=None):
        """Edit marks (docs/SPEC.md section 14): (added, removed, detail, line_base_old, line_base_new, dels, ins) - dels[g] = 1
        for every line g of `olds` the canonical script deletes, ins[g] = 1 for every line g of `news` it inserts (global line
        order of each side; line_base[i] = first line of file i).  Arrays too small for the lines are sized and the call made
        again (cap: the first guess)."""
        n = olds.n_files
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        bo, bn = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
        a, b = olds.c_struct(), news.c_struct()
        co = cn = int(cap if cap is not None else 0)
        for _ in range(2):
            dels, ins = np.zeros(max(co, 1), np.uint8), np.zeros(max(cn, 1), np.uint8)
            mk = _LineMarks(_p(bo), _p(bn), _p(dels), co, 0, _p(ins), cn, 0)
            rc = lib().tsm_diff_pairs_marks(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(mk), stream)
            if rc == TSM_E_CAPACITY and (mk.n_old > co or mk.n_new > cn):
                co, cn = int(mk.n_old), int(mk.n_new)
                continue
            if rc:
                raise TsmError(rc, "tsm_diff_pairs_marks")
            return added, removed, det[:n], bo, bn, dels[:mk.n_old], ins[:mk.n_new]
        raise TsmError(TSM_E_CAPACITY, "tsm_diff_pairs_marks")

    def diff_cases(self, olds, news, stream=None, cap=None):
        """Test-case churn (docs/SPEC.md section 16): (added, removed, detail, old_cases, new_cases) with the cases of every old
        and every new side as CASE arrays in global line order (pair, 0-based header line, lines, assertion lines, deleted or
        inserted lines, deleted or inserted assertion lines, and for new cases the index of the old case matched by its kept
        header line, else -1).  Arrays too small for the cases are sized and the call made again (cap: the first guess)."""
        n = olds.n_files
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        a, b = olds.c_struct(), news.c_struct()
        co = cn = int(cap if cap is not None else 0)
        for _ in range(2):
            oc, nc = np.zeros(max(co, 1), CASE), np.zeros(max(cn, 1), CASE)
            r = _DiffCases(_p(oc), co, 0, _p(nc), cn, 0)
            rc = lib().tsm_diff_pairs_cases(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(r), stream)
            if rc == TSM_E_CAPACITY and (r.n_old > co or r.n_new > cn):
                co, cn = int(r.n_old), int(r.n_new)
                continue
            if rc:
                raise TsmError(rc, "tsm_diff_pairs_cases")
            return added, removed, det[:n], oc[:r.n_old], nc[:r.n_new]
        raise TsmError(TSM_E_CAPACITY, "tsm_diff_pairs_cases")

    def diff_assert_edits(self, olds, news, stream=None, cap=None):
        """Assertion edits (docs/SPEC.md section 17): diff_pairs(asserts=True)'s (added, removed, detail, added_counts,
        removed_counts, added_events, removed_events) plus an ASSERT_EDIT array: per edit the index of the deleted line in
        removed_events (rev), of the inserted line in added_events (aev) and the score (similarity in % = score // 600),
        ordered by aev.  Arrays too small for the events or the edits are sized and the call made again (cap: the first guess
        for each)."""
        n = olds.n_files
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        a, b = olds.c_struct(), news.c_struct()
        ce = int(cap if cap is not None else (olds.source_bytes + news.source_bytes) // 1024 + 4096)
        ck = ce
        for _ in range(2):
            ac, rc_ = np.zeros((olds.n_groups, K), np.int64), np.zeros((olds.n_groups, K), np.int64)
            aev, rev, ed = np.zeros(max(ce, 1), ASSERT_EVENT), np.zeros(max(ce, 1), ASSERT_EVENT), np.zeros(max(ck, 1), ASSERT_EDIT)
            r = _DiffAsserts(_p(ac), _p(rc_), _p(aev), ce, 0, _p(rev), ce, 0)
            ne = C.c_int64(0)
            rc = lib().tsm_diff_pairs_assert_edits(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(r),
                                                   _p(ed), ck, C.byref(ne), stream)
            if rc == TSM_E_CAPACITY and (max(r.n_aev, r.n_rev) > ce or ne.value > ck):
                ce, ck = max(ce, int(r.n_aev), int(r.n_rev)), max(ck, int(ne.value))
                continue
            if rc:
                raise TsmError(rc, "tsm_diff_pairs_assert_edits")
            return added, removed, det[:n], ac, rc_, aev[:r.n_aev], rev[:r.n_rev], ed[:ne.value]
        raise TsmError(TSM_E_CAPACITY, "tsm_diff_pairs_assert_edits")

    def assert_edits_last_ms(self):
        """Phases of the last diff_assert_edits call in ms: [k_scan over both sides, the diff kernels, compact to pairing
        (host clock)]."""
        ms = (C.c_float * 3)()
        lib().tsm_assert_edits_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def blame_pairs(self, olds, news, prev, label, heads, stream=None, cap=None):
        """Line provenance (docs/SPEC.md section 14): (added, removed, detail, line_base_new, origins) with origins an ORIGIN array
        over every line of `news` (line_base_new[i] = first line of file i).  prev[i]: the pair whose new side is pair i's old
        side, or -1; heads: {pair: ORIGIN array of its old side's lines} for the pairs with prev -1 (a missing head has a file
        with no lines); label[i]: the change of the lines pair i inserts."""
        n = olds.n_files
        prev = np.ascontiguousarray(prev, np.int32)
        label = np.ascontiguousarray(label, np.int32)
        in_base = np.zeros(n + 1, np.int64)
        parts = []
        for i in range(n):
            h = heads.get(i) if prev[i] < 0 else None
            h = np.zeros(0, ORIGIN) if h is None else np.ascontiguousarray(h, ORIGIN)
            parts.append(h)
            in_base[i + 1] = in_base[i] + len(h)
        origin_in = np.concatenate(parts) if parts else np.zeros(0, ORIGIN)
        origin_in = origin_in if len(origin_in) else np.zeros(1, ORIGIN)
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        bo, bn = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
        a, b = olds.c_struct(), news.c_struct()
        c = int(cap if cap is not None else 0)
        for _ in range(2):
            out = np.zeros(max(c, 1), ORIGIN)
            nl = C.c_int64()
            rc = lib().tsm_blame_pairs(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), _p(prev), _p(label),
                                       _p(origin_in), _p(in_base), _p(bo), _p(bn), _p(out), c, C.byref(nl), stream)
            if rc == TSM_E_CAPACITY and nl.value > c:
                c = int(nl.value)
                continue
            if rc:
                raise TsmError(rc, "tsm_blame_pairs")
            return added, removed, det[:n], bn, out[:nl.value]
        raise TsmError(TSM_E_CAPACITY, "tsm_blame_pairs")

    def blame_last_ms(self):
        """Device time of k_blame in the last blame_pairs call, in ms."""
        ms = C.c_float()
        lib().tsm_blame_last_ms(self._ctx, C.byref(ms))
        return float(ms.value)

    def similarity(self, olds, news, cand_old, cand_new, stream=None):
        """Rename similarity (docs/SPEC.md section 13): common[c] of file cand_old[c] of `olds` and file cand_new[c] of `news`
        as np.int64[n_cand] (git's score is common * 60000 // max(size_old, size_new))."""
        co = np.ascontiguousarray(cand_old, np.int32).ravel()
        cn = np.ascontiguousarray(cand_new, np.int32).ravel()
        if co.size != cn.size:
            raise ValueError("cand_old and cand_new differ in length")
        out = np.zeros(max(co.size, 1), np.int64)
        a, b = olds.c_struct(), news.c_struct()
        rc = lib().tsm_similarity(self._ctx, C.byref(a), C.byref(b), _p(co), _p(cn), co.size, _p(out), stream)
        if rc:
            raise TsmError(rc, "tsm_similarity")
        return out[:co.size]

    def similarity_last_ms(self):
        """Device time of the last similarity call: [k_scan over both sides, sort / merge, k_similarity] in ms."""
        ms = (C.c_float * 3)()
        lib().tsm_similarity_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def clones(self, corpus, min_lines=5, blind=False, stream=None, cap=None):
        """Duplicated test code (docs/SPEC.md section 15): a dict of numpy arrays line_base[n_files+1], file_dup[n_files],
        file_dup_assert[n_files], class_base[n_classes+1], class_len[n_classes] and member[n_members] (the global first line of
        every fragment; class c is member[class_base[c]:class_base[c+1]], each fragment class_len[c] lines).  Arrays too small
        for the classes or fragments are sized from the counts and the call is made again (cap: the first guess of both).
        blind=True: the near-miss clones of section 21 (tsm_clones_blind) over the kept lines, member, class_len, file_dup and
        file_dup_assert in kept lines, plus kept_base[n_files+1], kept_line[n_kept] (the global line of every kept line),
        blind_hash[n_kept] and file_kept_assert[n_files]."""
        n = corpus.n_files
        cs = corpus.c_struct()
        cc = cm = ck = int(cap if cap is not None else 0)
        what = "tsm_clones_blind" if blind else "tsm_clones"
        for _ in range(2):
            out = {"line_base": np.zeros(n + 1, np.int64), "file_dup": np.zeros(n, np.uint32), "file_dup_assert": np.zeros(n, np.uint32),
                   "class_base": np.zeros(cc + 1, np.int64), "class_len": np.zeros(max(cc, 1), np.uint32),
                   "member": np.zeros(max(cm, 1), np.int64)}
            r = _CloneResult(*[_p(out[k]) for k in ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len")], cc, 0,
                             _p(out["member"]), cm, 0)
            if blind:
                out.update(kept_base=np.zeros(n + 1, np.int64), kept_line=np.zeros(max(ck, 1), np.int64),
                           blind_hash=np.zeros(max(ck, 1), np.uint64), file_kept_assert=np.zeros(n, np.uint32))
                b = _BlindResult(*[_p(out[k]) for k in ("kept_base", "kept_line", "blind_hash", "file_kept_assert")], ck, 0)
                rc = lib().tsm_clones_blind(self._ctx, C.byref(cs), int(min_lines), C.byref(b), C.byref(r), stream)
                short_kept = b.n_kept > ck
            else:
                rc = lib().tsm_clones(self._ctx, C.byref(cs), int(min_lines), C.byref(r), stream)
                short_kept = False
            if rc == TSM_E_CAPACITY and (r.n_classes > cc or r.n_members > cm or short_kept):
                cc, cm = int(r.n_classes), int(r.n_members)
                if blind:
                    ck = int(b.n_kept)
                continue
            if rc:
                raise TsmError(rc, what)
            out["class_base"] = out["class_base"][:r.n_classes + 1]
            out["class_len"] = out["class_len"][:r.n_classes]
            out["member"] = out["member"][:r.n_members]
            if blind:
                out["kept_line"], out["blind_hash"] = out["kept_line"][:b.n_kept], out["blind_hash"][:b.n_kept]
            return out
        raise TsmError(TSM_E_CAPACITY, what)

    def smells(self, corpus, stream=None, cap=None):
        """Test smells (docs/SPEC.md section 18): a dict of numpy arrays line_base[n_files+1], line_smell[n_lines] (the smell bits
        of every line: bit k is SMELLS[k]) and tests[n_tests] (SMELL_TEST records in global line order).  Arrays too small for
        the lines or tests are sized from the counts and the call is made again (cap: the first guess of both)."""
        n = corpus.n_files
        cs = corpus.c_struct()
        cl = ct = int(cap if cap is not None else 0)
        for _ in range(2):
            base = np.zeros(n + 1, np.int64)
            smell = np.zeros(max(cl, 1), np.uint16)
            tests = np.zeros(max(ct, 1), SMELL_TEST)
            nl, nt = C.c_int64(), C.c_int64()
            rc = lib().tsm_smells(self._ctx, C.byref(cs), _p(base), _p(smell), cl, C.byref(nl), _p(tests), ct, C.byref(nt), stream)
            if rc == TSM_E_CAPACITY and (nl.value > cl or nt.value > ct):
                cl, ct = int(nl.value), int(nt.value)
                continue
            if rc:
                raise TsmError(rc, "tsm_smells")
            return {"line_base": base, "line_smell": smell[:nl.value], "tests": tests[:nt.value]}
        raise TsmError(TSM_E_CAPACITY, "tsm_smells")

    def smells_lexical(self, corpus, stream=None, cap=None):
        """Test smells with the lexical smells (docs/SPEC.md section 25): the dict of smells() - line_base, line_smell and tests,
        exactly as smells() returns them - plus line_lsmell[n_lines] (bit k is LSMELLS[k]) and lex[n_tests] (LEX_TEST records,
        in the order of tests).  Arrays too small are sized from the counts and the call is made again (cap: the first guess)."""
        n = corpus.n_files
        cs = corpus.c_struct()
        cl = ct = int(cap if cap is not None else 0)
        for _ in range(2):
            base = np.zeros(n + 1, np.int64)
            smell, lsmell = np.zeros(max(cl, 1), np.uint16), np.zeros(max(cl, 1), np.uint8)
            tests, lex = np.zeros(max(ct, 1), SMELL_TEST), np.zeros(max(ct, 1), LEX_TEST)
            nl, nt = C.c_int64(), C.c_int64()
            rc = lib().tsm_smells_lexical(self._ctx, C.byref(cs), _p(base), _p(smell), _p(lsmell), cl, C.byref(nl), _p(tests), _p(lex),
                                          ct, C.byref(nt), stream)
            if rc == TSM_E_CAPACITY and (nl.value > cl or nt.value > ct):
                cl, ct = int(nl.value), int(nt.value)
                continue
            if rc:
                raise TsmError(rc, "tsm_smells_lexical")
            return {"line_base": base, "line_smell": smell[:nl.value], "tests": tests[:nt.value], "line_lsmell": lsmell[:nl.value],
                    "lex": lex[:nt.value]}
        raise TsmError(TSM_E_CAPACITY, "tsm_smells_lexical")

    def test_links(self, corpus, role, stem=None, stream=None, cap=None):
        """Test-to-code links (docs/SPEC.md section 27): a dict of tests (LINK_TEST, one per test of a test file), links (LINK, in
        (test, first call) order) and defs (LINK_DEF, one per definition of a production file).  role[f] != 0 marks a test file;
        stem[f] is focal_stems' id (None: no focal files).  Arrays too small are sized from the counts and the call is made again
        (cap: the first guess for every array)."""
        cs = corpus.c_struct()
        role = np.ascontiguousarray(role, np.uint8)
        stem = None if stem is None else np.ascontiguousarray(stem, np.int32)
        ct = ck = cd = int(cap if cap is not None else 0)
        for _ in range(2):
            tests, links, defs = np.zeros(max(ct, 1), LINK_TEST), np.zeros(max(ck, 1), LINK), np.zeros(max(cd, 1), LINK_DEF)
            r = _LinksResult(tests=_p(tests), test_cap=ct, links=_p(links), link_cap=ck, defs=_p(defs), def_cap=cd)
            rc = lib().tsm_test_links(self._ctx, C.byref(cs), _p(role), _p(stem), C.byref(r), stream)
            if rc == TSM_E_CAPACITY and (r.n_tests > ct or r.n_links > ck or r.n_defs > cd):
                ct, ck, cd = int(r.n_tests), int(r.n_links), int(r.n_defs)
                continue
            if rc:
                raise TsmError(rc, "tsm_test_links")
            return {"tests": tests[:r.n_tests], "links": links[:r.n_links], "defs": defs[:r.n_defs]}
        raise TsmError(TSM_E_CAPACITY, "tsm_test_links")

    def diff_smells(self, olds, news, stream=None, cap=None):
        """Test-smell churn (docs/SPEC.md section 19): a dict of added, removed, detail (tsm_diff_pairs_detail's), old_cases and
        new_cases (diff_cases' CASE arrays), old_tests and new_tests (SMELL_TEST records of each side, file = the pair) and
        old_churn and new_churn (one TEST_CHURN record per test: its case index, and per smell its instances and those that the
        revision removes (old side) or adds (new side)).  Arrays too small for the cases or tests are sized from the counts and
        the call is made again (cap: the first guess of each)."""
        n = olds.n_files
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        a, b = olds.c_struct(), news.c_struct()
        co = cn = to = tn = int(cap if cap is not None else 0)
        for _ in range(2):
            oc, nc = np.zeros(max(co, 1), CASE), np.zeros(max(cn, 1), CASE)
            ot, nt = np.zeros(max(to, 1), SMELL_TEST), np.zeros(max(tn, 1), SMELL_TEST)
            och, nch = np.zeros(max(to, 1), TEST_CHURN), np.zeros(max(tn, 1), TEST_CHURN)
            r = _DiffSmells(_DiffCases(_p(oc), co, 0, _p(nc), cn, 0), _p(ot), _p(och), to, 0, _p(nt), _p(nch), tn, 0)
            rc = lib().tsm_diff_pairs_smells(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(r), stream)
            k = r.cases
            if rc == TSM_E_CAPACITY and (k.n_old > co or k.n_new > cn or r.n_old_tests > to or r.n_new_tests > tn):
                co, cn, to, tn = int(k.n_old), int(k.n_new), int(r.n_old_tests), int(r.n_new_tests)
                continue
            if rc:
                raise TsmError(rc, "tsm_diff_pairs_smells")
            return {"added": added, "removed": removed, "detail": det[:n], "old_cases": oc[:k.n_old], "new_cases": nc[:k.n_new],
                    "old_tests": ot[:r.n_old_tests], "new_tests": nt[:r.n_new_tests], "old_churn": och[:r.n_old_tests],
                    "new_churn": nch[:r.n_new_tests]}
        raise TsmError(TSM_E_CAPACITY, "tsm_diff_pairs_smells")

    def diff_smells_lexical(self, olds, news, stream=None, cap=None):
        """Lexical test-smell churn (docs/SPEC.md section 26): the dict of diff_smells(), exactly as it returns it, plus old_lex and
        new_lex (LEX_TEST records of each side, in the order of its tests) and old_lex_churn and new_lex_churn (one LEX_CHURN
        record per test: per lexical smell its instances and those that the revision removes (old side) or adds (new side)).
        Arrays too small are sized from the counts and the call is made again (cap: the first guess of each)."""
        n = olds.n_files
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        a, b = olds.c_struct(), news.c_struct()
        co = cn = to = tn = int(cap if cap is not None else 0)
        for _ in range(2):
            oc, nc = np.zeros(max(co, 1), CASE), np.zeros(max(cn, 1), CASE)
            ot, nt = np.zeros(max(to, 1), SMELL_TEST), np.zeros(max(tn, 1), SMELL_TEST)
            och, nch = np.zeros(max(to, 1), TEST_CHURN), np.zeros(max(tn, 1), TEST_CHURN)
            ol, nl = np.zeros(max(to, 1), LEX_TEST), np.zeros(max(tn, 1), LEX_TEST)
            olc, nlc = np.zeros(max(to, 1), LEX_CHURN), np.zeros(max(tn, 1), LEX_CHURN)
            r = _DiffSmells(_DiffCases(_p(oc), co, 0, _p(nc), cn, 0), _p(ot), _p(och), to, 0, _p(nt), _p(nch), tn, 0)
            x = _DiffLexSmells(_p(ol), _p(olc), _p(nl), _p(nlc))
            rc = lib().tsm_diff_pairs_smells_lexical(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(r),
                                                     C.byref(x), stream)
            k = r.cases
            if rc == TSM_E_CAPACITY and (k.n_old > co or k.n_new > cn or r.n_old_tests > to or r.n_new_tests > tn):
                co, cn, to, tn = int(k.n_old), int(k.n_new), int(r.n_old_tests), int(r.n_new_tests)
                continue
            if rc:
                raise TsmError(rc, "tsm_diff_pairs_smells_lexical")
            return {"added": added, "removed": removed, "detail": det[:n], "old_cases": oc[:k.n_old], "new_cases": nc[:k.n_new],
                    "old_tests": ot[:r.n_old_tests], "new_tests": nt[:r.n_new_tests], "old_churn": och[:r.n_old_tests],
                    "new_churn": nch[:r.n_new_tests], "old_lex": ol[:r.n_old_tests], "new_lex": nl[:r.n_new_tests],
                    "old_lex_churn": olc[:r.n_old_tests], "new_lex_churn": nlc[:r.n_new_tests]}
        raise TsmError(TSM_E_CAPACITY, "tsm_diff_pairs_smells_lexical")

    def diff_smells_lexical_last_ms(self):
        """Device time of the last diff_smells_lexical call: [k_scan over both sides, smell and lexical stages, the diff, case
        records + k_smell_churn] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_diff_smells_lexical_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def diff_smells_last_ms(self):
        """Device time of the last diff_smells call: [k_scan over both sides, smell stages, the diff, case records +
        k_smell_churn] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_diff_smells_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def diff_moves(self, olds, news, stream=None, cap=None):
        """Moved code (docs/SPEC.md section 20): a dict of added, removed, detail (tsm_diff_pairs_detail's), line_base_old and
        line_base_new, dels and ins (diff_marks' marks with bit 1 set on every moved line, so a moved line is 3) and old_blocks and
        new_blocks (MOVE_BLOCK arrays in line order: global first line, the partner's global line on the other side, lines and
        assertion lines).  A pair's step is its grp: olds and news must carry the same grp per pair.  Arrays too small for the
        lines or blocks are sized from the counts and the call is made again (cap: the first guess of each)."""
        n = olds.n_files
        added, removed, det = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(max(n, 1), DIFF_DETAIL)
        bo, bn = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
        a, b = olds.c_struct(), news.c_struct()
        co = cn = bko = bkn = int(cap if cap is not None else 0)
        for _ in range(2):
            dels, ins = np.zeros(max(co, 1), np.uint8), np.zeros(max(cn, 1), np.uint8)
            ob, nb = np.zeros(max(bko, 1), MOVE_BLOCK), np.zeros(max(bkn, 1), MOVE_BLOCK)
            r = _DiffMoves(_LineMarks(_p(bo), _p(bn), _p(dels), co, 0, _p(ins), cn, 0), _p(ob), bko, 0, _p(nb), bkn, 0)
            rc = lib().tsm_diff_pairs_moves(self._ctx, C.byref(a), C.byref(b), _p(added), _p(removed), _p(det), C.byref(r), stream)
            mk = r.marks
            if rc == TSM_E_CAPACITY and (mk.n_old > co or mk.n_new > cn or r.n_old_blocks > bko or r.n_new_blocks > bkn):
                co, cn, bko, bkn = int(mk.n_old), int(mk.n_new), int(r.n_old_blocks), int(r.n_new_blocks)
                continue
            if rc:
                raise TsmError(rc, "tsm_diff_pairs_moves")
            return {"added": added, "removed": removed, "detail": det[:n], "line_base_old": bo, "line_base_new": bn,
                    "dels": dels[:mk.n_old], "ins": ins[:mk.n_new], "old_blocks": ob[:r.n_old_blocks], "new_blocks": nb[:r.n_new_blocks]}
        raise TsmError(TSM_E_CAPACITY, "tsm_diff_pairs_moves")

    def moves_last_ms(self):
        """Device time of the last diff_moves call: [k_scan over both sides, the diff, line flags + join + k_move_reach,
        k_move_starts + k_move_runs + k_move_mark] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_moves_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def similar_tests(self, corpus, min_lines=5, similarity=70, stream=None, cap=None):
        """Similar tests (docs/SPEC.md section 23): a dict of numpy arrays tests[n_tests] (SMELL_TEST, as smells() gives them),
        test_kept[n_tests] (kept blind lines of each test), pairs[n_pairs] (SIMILAR_PAIR, ascending (a, b)), class_base[n_classes+1]
        and member[n_members] (test indices), and n_candidates (the pairs whose LCS was computed).  Arrays too small for their
        counts are sized from the counts and the call is made again, which repeats the whole all-pairs work.  By default the tests,
        members and classes are sized from the corpus' line count (a test starts on a line), so only more pairs than that guess
        (at least 2^16, at most 2^22) cause a second call; cap: the first guess of every array instead."""
        cs = corpus.c_struct()
        if cap is None:
            lines = int(np.count_nonzero(np.asarray(corpus.arena[:int(corpus.off[corpus.n_files])]) == 0x0A)) + corpus.n_files
            ct = cc = cm = lines
            cp = min(max(4 * lines, 1 << 16), 1 << 22)
        else:
            ct = cp = cc = cm = int(cap)
        for _ in range(2):
            tests, kept = np.zeros(max(ct, 1), SMELL_TEST), np.zeros(max(ct, 1), np.uint32)
            pairs = np.zeros(max(cp, 1), SIMILAR_PAIR)
            cbase, member = np.zeros(cc + 1, np.int64), np.zeros(max(cm, 1), np.int32)
            r = _SimilarResult(_p(tests), _p(kept), ct, 0, _p(pairs), cp, 0, _p(cbase), cc, 0, _p(member), cm, 0, 0)
            rc = lib().tsm_similar_tests(self._ctx, C.byref(cs), int(min_lines), int(similarity), C.byref(r), stream)
            if rc == TSM_E_CAPACITY and (r.n_tests > ct or r.n_pairs > cp or r.n_classes > cc or r.n_members > cm):
                ct, cp, cc, cm = int(r.n_tests), int(r.n_pairs), int(r.n_classes), int(r.n_members)
                continue
            if rc:
                raise TsmError(rc, "tsm_similar_tests")
            return {"tests": tests[:r.n_tests], "test_kept": kept[:r.n_tests], "pairs": pairs[:r.n_pairs],
                    "class_base": cbase[:r.n_classes + 1], "member": member[:r.n_members], "n_candidates": int(r.n_candidates)}
        raise TsmError(TSM_E_CAPACITY, "tsm_similar_tests")

    def similar_tests_last_ms(self):
        """Device time of the last similar_tests call: [k_scan, case spans + smell stage + lexer, tokens + posting lists +
        enumeration, verification] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_similar_tests_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def similar_churn(self, old_rev, new_rev, pair_old, pair_new, min_lines=5, similarity=70, stream=None, cap=None):
        """Similar-test churn (docs/SPEC.md section 24): a dict {"old": ..., "new": ..., "events": ...}.  Per revision tests
        (SMELL_TEST, as similar_tests gives them), test_kept, match (the other side's test, -1 for none), change (b"A", b"D",
        b"=" or b"M" per test, as uint8) and n_candidates; events (SIMILAR_EVENT, status indexing SIMILAR_STATUSES).  Pair k
        is file pair_old[k] of old_rev and file pair_new[k] of new_rev, -1 for none; a file in no pair is unchanged and
        matches the same-numbered unpaired file of the other revision.  Arrays too small for their counts are sized from
        the counts and the call is made again, which repeats the whole call (cap: the first guess of each; by default the tests
        of each revision are sized from its line count and the events from both, at least 2^16 and at most 2^22)."""
        po = np.ascontiguousarray(pair_old, np.int32).ravel()
        pn = np.ascontiguousarray(pair_new, np.int32).ravel()
        if po.size != pn.size:
            raise ValueError("pair_old and pair_new differ in length")
        revs = (old_rev, new_rev)
        cs = [r.c_struct() for r in revs]
        if cap is None:
            caps = [int(np.count_nonzero(np.asarray(r.arena[:int(r.off[r.n_files])]) == 0x0A)) + r.n_files for r in revs]
            ce = min(max(sum(caps), 1 << 16), 1 << 22)
        else:
            caps, ce = [int(cap)] * 2, int(cap)
        for _ in range(2):
            outs, sides = [], []
            for ct in caps:
                o = {"tests": np.zeros(max(ct, 1), SMELL_TEST), "test_kept": np.zeros(max(ct, 1), np.uint32),
                     "match": np.zeros(max(ct, 1), np.int32), "change": np.zeros(max(ct, 1), np.uint8)}
                outs.append(o)
                sides.append(_SimilarChurnSide(*[_p(o[k]) for k in ("tests", "test_kept", "match", "change")], ct, 0, 0))
            ev = np.zeros(max(ce, 1), SIMILAR_EVENT)
            ne = C.c_int64()
            rc = lib().tsm_similar_churn(self._ctx, C.byref(cs[0]), C.byref(cs[1]), _p(po), _p(pn), po.size, int(min_lines), int(similarity),
                                         C.byref(sides[0]), C.byref(sides[1]), _p(ev), ce, C.byref(ne), stream)
            need = [int(sd.n_tests) for sd in sides]
            if rc == TSM_E_CAPACITY and (ne.value > ce or any(w > h for w, h in zip(need, caps))):
                caps, ce = need, int(ne.value)
                continue
            if rc:
                raise TsmError(rc, "tsm_similar_churn")
            res = {"events": ev[:ne.value]}
            for name, o, sd in zip(("old", "new"), outs, sides):
                res[name] = {k: v[:sd.n_tests] for k, v in o.items()}
                res[name]["n_candidates"] = int(sd.n_candidates)
            return res
        raise TsmError(TSM_E_CAPACITY, "tsm_similar_churn")

    def similar_churn_last_ms(self):
        """Device time of the last similar_churn call: [k_scan over both revisions, fronts of both + the marks diff +
        k_sc_change, tokens + posting lists + restricted enumeration, verification (cross scores included)] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_similar_churn_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def smells_last_ms(self):
        """Device time of the last smells call: [k_scan, kinds + case spans, k_smell_lines, k_smell_tests] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_smells_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def smells_lexical_last_ms(self):
        """Device time of the last smells_lexical call: [k_scan, the front (kinds, case spans, smell stage), lexer
        states + k_lex_body + k_lex_lines, k_lex_tests] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_smells_lexical_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def link_churn(self, old_rev, new_rev, old_role, new_role, pair_old, pair_new, old_stem=None, new_stem=None, stream=None,
                   cap=None):
        """Test-to-code link churn (docs/SPEC.md section 28): a dict {"old": ..., "new": ..., "events": ...}.  Per revision tests,
        links and defs (as test_links gives them for that revision alone, as one repository), match (the other side's link test,
        -1 for none) and change (b"A", b"D", b"=" or b"M" per link test, as uint8); events (LINK_EVENT, event indexing LINK_EVENTS
        and cause LINK_CAUSES).  role and stem per revision are those of test_links.  Pair k is file pair_old[k] of old_rev and
        file pair_new[k] of new_rev, -1 for none; a file in no pair is unchanged and matches the same-numbered unpaired file of
        the other revision.  Arrays too small for their counts are sized from the counts and the call is made again, which
        repeats the whole call (cap: the first guess of every array)."""
        po = np.ascontiguousarray(pair_old, np.int32).ravel()
        pn = np.ascontiguousarray(pair_new, np.int32).ravel()
        if po.size != pn.size:
            raise ValueError("pair_old and pair_new differ in length")
        cs = [old_rev.c_struct(), new_rev.c_struct()]
        roles = [np.ascontiguousarray(old_role, np.uint8), np.ascontiguousarray(new_role, np.uint8)]
        stems = [None if s is None else np.ascontiguousarray(s, np.int32) for s in (old_stem, new_stem)]
        caps = [[int(cap if cap is not None else 0)] * 3 for _ in range(2)]
        ce = int(cap if cap is not None else 0)
        for _ in range(2):
            outs, sides = [], []
            for ct, ck, cd in caps:
                o = {"tests": np.zeros(max(ct, 1), LINK_TEST), "links": np.zeros(max(ck, 1), LINK), "defs": np.zeros(max(cd, 1), LINK_DEF),
                     "match": np.zeros(max(ct, 1), np.int32), "change": np.zeros(max(ct, 1), np.uint8)}
                outs.append(o)
                r = _LinksResult(tests=_p(o["tests"]), test_cap=ct, links=_p(o["links"]), link_cap=ck, defs=_p(o["defs"]), def_cap=cd)
                sides.append(_LinkChurnSide(r, _p(o["match"]), _p(o["change"])))
            ev = np.zeros(max(ce, 1), LINK_EVENT)
            ne = C.c_int64()
            rc = lib().tsm_link_churn(self._ctx, C.byref(cs[0]), C.byref(cs[1]), _p(roles[0]), _p(stems[0]), _p(roles[1]), _p(stems[1]),
                                      _p(po), _p(pn), po.size, C.byref(sides[0]), C.byref(sides[1]), _p(ev), ce, C.byref(ne), stream)
            need = [[int(sd.links.n_tests), int(sd.links.n_links), int(sd.links.n_defs)] for sd in sides]
            if rc == TSM_E_CAPACITY and (ne.value > ce or any(w > h for nw, nh in zip(need, caps) for w, h in zip(nw, nh))):
                caps, ce = need, int(ne.value)
                continue
            if rc:
                raise TsmError(rc, "tsm_link_churn")
            res = {"events": ev[:ne.value]}
            for name, o, sd in zip(("old", "new"), outs, sides):
                nt = int(sd.links.n_tests)
                res[name] = {"tests": o["tests"][:nt], "links": o["links"][:sd.links.n_links], "defs": o["defs"][:sd.links.n_defs],
                             "match": o["match"][:nt], "change": o["change"][:nt]}
            return res
        raise TsmError(TSM_E_CAPACITY, "tsm_link_churn")

    def link_churn_last_ms(self):
        """Device time of the last link_churn call: [k_scan over both revisions, both link fronts + the marks diff +
        k_lc_change, both link joins, the churn join and emit] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_link_churn_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def test_links_last_ms(self):
        """Device time of the last test_links call: [k_scan, the front (kinds, case spans, smell stage, lexer states, the tests
        of the test files and their code lines), k_link_lines, the join to the records] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_test_links_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def clones_last_ms(self):
        """Device time of the last clones call: [k_scan, grouping + classes, members + coverage] in ms."""
        ms = (C.c_float * 3)()
        lib().tsm_clones_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def clones_blind_last_ms(self):
        """Device time of the last clones call with blind=True: [k_scan, lexing + compaction, grouping + classes, members +
        coverage] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_clones_blind_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]

    def clone_churn(self, old_rev, new_rev, pair_old, pair_new, min_lines=5, blind=False, stream=None, cap=None):
        """Clone churn (docs/SPEC.md section 22): a dict {"old": ..., "new": ...}, per revision the dict of clones(rev, min_lines,
        blind) for that revision alone plus per fragment changed, changed_assert and state (FRAG_STATES) and per class
        class_counts[n_classes, 3] (kept, edited, whole fragments) and status (CLONE_STATUSES).  Pair k is file pair_old[k] of
        old_rev and file pair_new[k] of new_rev, -1 for none.  Arrays too small for the classes, fragments or kept lines are sized
        from the counts and the call is made again (cap: the first guess of each)."""
        po = np.ascontiguousarray(pair_old, np.int32).ravel()
        pn = np.ascontiguousarray(pair_new, np.int32).ravel()
        if po.size != pn.size:
            raise ValueError("pair_old and pair_new differ in length")
        revs = (old_rev, new_rev)
        cs = [r.c_struct() for r in revs]
        g = int(cap if cap is not None else 0)
        caps = [[g, g, g], [g, g, g]]                       # per side: classes, fragments, kept lines
        for _ in range(2):
            outs, sides = [], []
            for r, (cc, cm, ck) in zip(revs, caps):
                n = r.n_files
                o = {"line_base": np.zeros(n + 1, np.int64), "file_dup": np.zeros(n, np.uint32), "file_dup_assert": np.zeros(n, np.uint32),
                     "class_base": np.zeros(cc + 1, np.int64), "class_len": np.zeros(max(cc, 1), np.uint32),
                     "member": np.zeros(max(cm, 1), np.int64), "changed": np.zeros(max(cm, 1), np.uint32),
                     "changed_assert": np.zeros(max(cm, 1), np.uint32), "state": np.zeros(max(cm, 1), np.uint8),
                     "class_counts": np.zeros((max(cc, 1), 3), np.uint32), "status": np.zeros(max(cc, 1), np.uint8)}
                cr = _CloneResult(*[_p(o[k]) for k in ("line_base", "file_dup", "file_dup_assert", "class_base", "class_len")], cc, 0,
                                  _p(o["member"]), cm, 0)
                br = _BlindResult(None, None, None, None, 0, 0)
                if blind:
                    o.update(kept_base=np.zeros(n + 1, np.int64), kept_line=np.zeros(max(ck, 1), np.int64),
                             blind_hash=np.zeros(max(ck, 1), np.uint64), file_kept_assert=np.zeros(n, np.uint32))
                    br = _BlindResult(*[_p(o[k]) for k in ("kept_base", "kept_line", "blind_hash", "file_kept_assert")], ck, 0)
                outs.append(o)
                sides.append(_CloneChurnSide(cr, br, *[_p(o[k]) for k in ("changed", "changed_assert", "state", "class_counts", "status")]))
            rc = lib().tsm_clone_churn(self._ctx, C.byref(cs[0]), C.byref(cs[1]), _p(po), _p(pn), po.size, int(min_lines), int(bool(blind)),
                                       C.byref(sides[0]), C.byref(sides[1]), stream)
            need = [[int(sd.clones.n_classes), int(sd.clones.n_members), int(sd.blind.n_kept) if blind else 0] for sd in sides]
            if rc == TSM_E_CAPACITY and any(w > h for nd, cp in zip(need, caps) for w, h in zip(nd, cp)):
                caps = need
                continue
            if rc:
                raise TsmError(rc, "tsm_clone_churn")
            res = {}
            for name, o, (nc, nm, nk) in zip(("old", "new"), outs, need):
                for k in ("class_len", "class_counts", "status"):
                    o[k] = o[k][:nc]
                o["class_base"] = o["class_base"][:nc + 1]
                for k in ("member", "changed", "changed_assert", "state"):
                    o[k] = o[k][:nm]
                if blind:
                    o["kept_line"], o["blind_hash"] = o["kept_line"][:nk], o["blind_hash"][:nk]
                res[name] = o
            return res
        raise TsmError(TSM_E_CAPACITY, "tsm_clone_churn")

    def clone_churn_last_ms(self):
        """Device time of the last clone_churn call: [k_scan over both revisions, classes of both, k_churn_gather + the marks
        diff, k_churn_marks + the churn kernels of both sides] in ms."""
        ms = (C.c_float * 4)()
        lib().tsm_clone_churn_last_ms(self._ctx, C.byref(ms))
        return [float(x) for x in ms]
