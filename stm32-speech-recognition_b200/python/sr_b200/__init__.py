"""ctypes binding of libspeech_b200.so (include/speech_recog.h, include/sr_synth.h).

Plumbing for tests/ and bench.py only -- the product is the C-ABI library itself. Nothing here
computes: every call forwards to the CUDA kernels and raises if the library or a GPU is missing
(there is no CPU fallback). Struct layouts mirror the reference's VAD.H:10-22 / MFCC.H:18-25.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PKG_ROOT = os.path.normpath(os.path.join(_HERE, "..", ".."))
LIB_PATH = os.path.join(PKG_ROOT, "lib", "libspeech_b200.so")

FRAME_LEN, FRAME_MOV, MFCC_NUM, VV_FRM_MAX = 160, 80, 12, 119
FTR_BYTES = 2860
SEG_NULL = 0xFFFFFFFF
DIS_ERR = 0xFFFFFFFF
SAVE_MASK = 12345
FTR_PER_COMM = 4               # SR_FTR_PER_COMM: bank slots per command
DTW_CHECK_SIGN, DTW_BAND, DTW_SYM_P1, DTW_ANY_RATE = 1, 2, 4, 8
DTW_LIFTER = 1 << 13           # SR_DTW_LIFTER: score liftered rows, a' = sat16(trunc(a * DTW_LIFTER_W[c] / 16))
DTW_LIFTER_W = (10, 16, 21, 25, 27, 28, 27, 25, 21, 16, 10, 4)   # SR_DTW_LIFTER_W
ST_OK, ST_VAD_FAIL, ST_MFCC_FAIL, ST_REJECT = 0, 1, 2, 3


def dtw_reject(q):
    """SR_DTW_REJECT(q): the runner-up margin rule of q per mille (0 = no rule), OR'ed into set_match's flags"""
    q = int(q)
    if not 0 <= q <= 0xFFFF:
        raise ValueError("margin %d per mille outside 0..65535" % q)
    return q << 16


def dtw_knn(k):
    """SR_DTW_KNN(k): decide by the mean of each command's k best template scores, 1 <= k <= 4 (0 = no rule), OR'ed
    into set_match's flags"""
    k = int(k)
    if not 0 <= k <= FTR_PER_COMM:
        raise ValueError("k = %d outside 0..%d" % (k, FTR_PER_COMM))
    return k << 8

PATH_MAX = 237                 # SR_PATH_MAX: the longest warping path, 2 * VV_FRM_MAX - 1 points

ATAP_DTYPE = np.dtype([("mid_val", "<u4"), ("n_thl", "<u2"), ("z_thl", "<u2"), ("s_thl", "<u4")])
FTR_DTYPE = np.dtype([("save_sign", "<u2"), ("frm_num", "<u2"), ("mfcc_dat", "<i2", (VV_FRM_MAX * MFCC_NUM,))])
assert ATAP_DTYPE.itemsize == 12 and FTR_DTYPE.itemsize == FTR_BYTES


RECOG_FIELDS = ("atap", "seg_off", "ftr", "score", "best_idx", "best_dis", "cmd", "status")


class RecogOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in RECOG_FIELDS]


def _recog_out(ptrs):
    """sr_recog_out of the fields in `ptrs` (numpy arrays or device pointers); the others are NULL"""
    return RecogOut(*[_p(ptrs.get(k)) for k in RECOG_FIELDS])


def _recog_arrays(B, T, want):
    """zeroed host arrays for the fields of sr_recog_out named in `want`, for B utterances and T templates"""
    shape = {"atap": (B, ATAP_DTYPE), "seg_off": ((B, 3, 2), np.uint32), "ftr": (B, FTR_DTYPE), "score": ((B, T), np.uint32),
             "best_idx": (B, np.uint32), "best_dis": (B, np.uint32), "cmd": (B, np.uint32), "status": (B, np.uint8)}
    return {k: np.zeros(*shape[k]) for k in RECOG_FIELDS if k in want}


CONN_FRM_MAX = 818             # SR_CONN_FRM_MAX: frames of a 65 535-sample segment
CONN_SLOT_MAX = 128            # SR_CONN_SLOT_MAX: the widest bank of the connected-word decoder
WORD_DTYPE = np.dtype([(k, "<u4") for k in ("slot", "cmd", "segment", "start", "end", "dis")])   # sr_conn_word
CONN_FIELDS = ("atap", "seg_off", "frm_num", "n_words", "words", "total", "status")


class ConnOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in CONN_FIELDS]


GRAM_STATE_MAX = 16            # SR_GRAM_STATE_MAX
GRAM_COPY_MAX = 128            # SR_GRAM_COPY_MAX


class GramArc(C.Structure):
    _fields_ = [("from_", C.c_uint32), ("to", C.c_uint32), ("cmd_mask", C.c_uint32)]


class Grammar(C.Structure):
    _fields_ = [("n_states", C.c_uint32), ("final_mask", C.c_uint32), ("n_arcs", C.c_uint32), ("arcs", C.POINTER(GramArc))]


def grammar(g):
    """(n_states, final_mask, [(from, to, cmd_mask), ...]) -> an sr_grammar (its arcs kept alive on the struct); a Grammar
    passes through, None stays None (NULL)"""
    if g is None or isinstance(g, Grammar):
        return g
    n_states, final_mask, arcs = g
    arr = (GramArc * max(len(arcs), 1))(*[GramArc(*a) for a in arcs])
    out = Grammar(n_states, final_mask, len(arcs), C.cast(arr, C.POINTER(GramArc)))
    out._arcs = arr
    return out


def loop_grammar(n_cmd=32):
    """the one-state loop grammar: any command, any number of times (exactly sr_connected_batch)"""
    return (1, 1, [(0, 0, (1 << n_cmd) - 1 if n_cmd < 32 else 0xFFFFFFFF)])


def chain_grammar(L, cmd_mask=0x3FF):
    """exactly L words, each a command of cmd_mask (default the ten digits): states 0..L, arcs k -> k+1, final state L"""
    return (L + 1, 1 << L, [(k, k + 1, cmd_mask) for k in range(L)])


LONG_U_MAX = 1 << 27           # SR_LONG_U_MAX: the longest recording of the long-form calls (include/sr_long.h)
LONG_SEG_DTYPE = np.dtype([(k, "<u4") for k in ("start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")])


class LongOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in ("atap", "n_segs", "segs")]


LONG_GRAM_FRM_MAX = 1677720    # SR_LONG_GRAM_FRM_MAX: frames of a 2^27-sample recording (include/sr_long_grammar.h)
LONG_GRAM_FIELDS = ("atap", "n_segs", "seg_off", "frm_num", "seg_status", "n_words", "words", "total")


class LongGramOut(C.Structure):
    _fields_ = [(k, C.c_void_p) for k in LONG_GRAM_FIELDS]


class StreamEvent(C.Structure):
    _fields_ = [(k, C.c_uint32) for k in ("stream", "segment", "start", "end", "status", "frm_num", "best_idx", "best_dis", "cmd")]


class ValidTag(C.Structure):
    _fields_ = [("start", C.c_void_p), ("end", C.c_void_p)]


_lib = None


def lib():
    """The loaded shared library (raises if it has not been built: run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libspeech_b200.so is not built (%s); run __graft_entry__.build()" % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int
        L.sr_create.argtypes = [i32, C.POINTER(vp)]
        L.sr_destroy.argtypes = [vp]
        L.sr_set_stream.argtypes = [vp, vp]
        L.sr_use_own_stream.argtypes = [vp]
        L.sr_sync.argtypes = [vp]
        L.sr_last_error.argtypes = [vp]
        L.sr_last_error.restype = C.c_char_p
        L.sr_host_alloc.argtypes = [C.c_size_t]
        L.sr_host_alloc.restype = vp
        L.sr_host_free.argtypes = [vp]
        L.sr_launch_count.argtypes = [vp]
        L.sr_launch_count.restype = u64
        L.sr_timing_enable.argtypes = [vp, u32]
        L.sr_timing_collect.argtypes = [vp, vp, vp, u32, vp]
        L.sr_debug_sqrt_mismatches.argtypes = [vp, u32, u32, vp]
        L.sr_debug_log100_mismatches.argtypes = [vp, u64, u64, vp]
        L.sr_debug_mag10_mismatches.argtypes = [vp, C.c_int, u64, u64, vp]
        L.sr_set_transport.argtypes = [vp, C.c_int]
        L.sr_transport_stats.argtypes = [vp, vp, vp, vp]
        L.sr_debug_pack12_host.argtypes = [C.c_int, vp, u64, vp]
        L.sr_debug_pack12_host.restype = u32
        L.sr_debug_unpack12.argtypes = [vp, vp, u64, vp]
        L.sr_enrol_batch.argtypes = [vp, vp, u32, u32, u32, vp, u32, vp]
        L.sr_get_mdl_batch.argtypes = [vp, vp, vp, u32, vp, vp]
        L.sr_dtw_path_batch.argtypes = [vp, vp, vp, u32, i32, vp, vp, vp]
        L.sr_average_bank.argtypes = [vp, vp, u32, u32, u32, i32, u32, vp, vp, vp]
        L.sr_mfcc_long_batch.argtypes = [vp, vp, u32, u32, vp, u32, vp, u32, vp, vp]
        L.sr_connected_batch.argtypes = [vp, vp, vp, u32, u32, u32, u32, vp, vp, vp]
        L.sr_recognise_connected_batch.argtypes = [vp, vp, u32, u32, u32, u32, u32, C.POINTER(ConnOut)]
        L.sr_connected_grammar_batch.argtypes = [vp, vp, vp, u32, u32, vp, u32, u32, vp, vp, vp]
        L.sr_recognise_connected_grammar_batch.argtypes = [vp, vp, u32, u32, u32, vp, u32, u32, C.POINTER(ConnOut)]
        L.sr_vad_long_batch.argtypes = [vp, vp, u32, u32, vp, u32, u32, vp, vp, vp]
        L.sr_vad_long_batch_dev.argtypes = [vp, vp, u32, u32, vp, u32, u32, vp, vp, vp]
        L.sr_recognise_long_batch.argtypes = [vp, vp, u32, u32, vp, u32, u32, C.POINTER(LongOut)]
        L.sr_recognise_long_batch_dev.argtypes = [vp, vp, u32, u32, vp, u32, u32, C.POINTER(LongOut)]
        L.sr_connected_grammar_segs_batch.argtypes = [vp, vp, vp, vp, u32, vp, u32, u32, vp, vp, vp]
        L.sr_recognise_long_grammar_batch.argtypes = [vp, vp, u32, u32, vp, u32, vp, u32, u32, u32, C.POINTER(LongGramOut)]
        L.sr_recognise_long_batch_at_rate.argtypes = [vp, vp, u32, u32, vp, u32, u32, u32, C.POINTER(LongOut)]
        L.sr_recognise_long_grammar_batch_at_rate.argtypes = [vp, vp, u32, u32, vp, u32, u32, vp, u32, u32, u32,
                                                              C.POINTER(LongGramOut)]
        L.sr_streams_create.argtypes = [vp, u32, u32, u32, C.POINTER(vp)]
        L.sr_streams_destroy.argtypes = [vp]
        L.sr_streams_reset.argtypes = [vp]
        L.sr_streams_push.argtypes = [vp, vp, u32, u32, vp, u32, vp]
        L.sr_streams_segments.argtypes = [vp, vp, vp]
        L.sr_streams_push_ragged.argtypes = [vp, vp, u32, vp, vp, u32, vp]
        L.sr_streams_fetch.argtypes = [vp, vp, u32, vp]
        L.sr_streams_pending.argtypes = [vp]
        L.sr_streams_pending.restype = u32
        L.sr_long_streams_create.argtypes = [vp, u32, u32, u32, vp, C.POINTER(vp)]
        L.sr_long_streams_create_at_rate.argtypes = [vp, u32, u32, u32, vp, u32, C.POINTER(vp)]
        L.sr_long_streams_destroy.argtypes = [vp]
        L.sr_long_streams_reset.argtypes = [vp, vp, vp]
        L.sr_long_streams_push.argtypes = [vp, vp, u32, u32, vp, u32, vp]
        L.sr_long_streams_push_ragged.argtypes = [vp, vp, u32, vp, vp, u32, vp]
        L.sr_long_streams_fetch.argtypes = [vp, vp, u32, vp]
        L.sr_long_streams_pending.argtypes = [vp]
        L.sr_long_streams_pending.restype = u32
        L.sr_long_streams_max_events.argtypes = [vp]
        L.sr_long_streams_max_events.restype = u32
        L.sr_long_streams_state.argtypes = [vp, vp, vp, vp, vp]
        L.sr_long_streams_ring_len.argtypes = [vp]
        L.sr_long_streams_ring_len.restype = u32
        L.sr_stream_group_create.argtypes = [C.POINTER(vp), u32, u32, u32, u32, C.POINTER(vp)]
        L.sr_streams_create_at_rate.argtypes = [vp, u32, u32, u32, u32, C.POINTER(vp)]
        L.sr_stream_group_create_at_rate.argtypes = [C.POINTER(vp), u32, u32, u32, u32, u32, C.POINTER(vp)]
        L.sr_stream_group_destroy.argtypes = [vp]
        L.sr_stream_group_reset.argtypes = [vp]
        L.sr_stream_group_push.argtypes = [vp, vp, u32, u32, vp, u32, vp]
        L.sr_stream_group_push_ragged.argtypes = [vp, vp, u32, vp, vp, u32, vp]
        L.sr_stream_group_segments.argtypes = [vp, vp, vp]
        L.sr_host_alloc_dev.argtypes = [i32, C.c_size_t]
        L.sr_host_alloc_dev.restype = vp
        L.sr_bind_thread_to_device.argtypes = [i32]
        L.sr_device_numa_node.argtypes = [i32]
        L.sr_host_numa_node.argtypes = [vp]
        L.sr_comm_unique_id.argtypes = [vp]
        L.sr_comm_create.argtypes = [vp, i32, i32, vp]
        L.sr_comm_destroy.argtypes = [vp]
        L.sr_comm_wait.argtypes = [vp]
        L.sr_allgather_dev.argtypes = [vp, vp, vp, C.c_size_t]
        L.sr_recognise_batch_dev_allgather.argtypes = [vp, vp, u32, u32, u32, C.POINTER(RecogOut), vp, vp]
        L.sr_set_dtw_variant.argtypes = [vp, i32]
        L.sr_set_match.argtypes = [vp, u32, i32]
        L.sr_get_match.argtypes = [vp, vp, vp]
        L.sr_set_geometry.argtypes = [vp, i32]
        L.sr_get_geometry.argtypes = [vp]
        L.sr_set_labels.argtypes = [vp, vp, u32, u32]
        L.sr_label.argtypes = [vp, u32]
        L.sr_label.restype = vp
        L.sr_set_bank.argtypes = [vp, vp, u32, u32]
        L.sr_set_bank_dev.argtypes = [vp, vp, u32, u32]
        for name in ("sr_noise_atap_batch", "sr_noise_atap_batch_dev"):
            getattr(L, name).argtypes = [vp, vp, u32, u32, u32, vp]
        for name in ("sr_vad_batch", "sr_vad_batch_dev"):
            getattr(L, name).argtypes = [vp, vp, u32, u32, u32, vp, vp]
        for name in ("sr_mfcc_batch", "sr_mfcc_batch_dev"):
            getattr(L, name).argtypes = [vp, vp, u32, u32, vp, u32, vp, vp]
        for name in ("sr_dtw_batch", "sr_dtw_batch_dev"):
            getattr(L, name).argtypes = [vp, vp, u32, u32, i32, vp, vp, vp]
        for name in ("sr_recognise_batch", "sr_recognise_batch_dev"):
            getattr(L, name).argtypes = [vp, vp, u32, u32, u32, C.POINTER(RecogOut)]
        L.sr_recognise_batch_multi.argtypes = [C.POINTER(vp), u32, vp, u32, u32, u32, C.POINTER(RecogOut)]
        L.sr_recognise_batch_at_rate.argtypes = [vp, vp, u32, u32, u32, u32, C.POINTER(RecogOut)]
        L.sr_recognise_batch_multi_at_rate.argtypes = [C.POINTER(vp), u32, vp, u32, u32, u32, u32, C.POINTER(RecogOut)]
        L.sr_enrol_batch_at_rate.argtypes = [vp, vp, u32, u32, u32, u32, vp, u32, vp]
        L.sr_recognise_connected_batch_at_rate.argtypes = [vp, vp, u32, u32, u32, u32, u32, u32, C.POINTER(ConnOut)]
        L.sr_recognise_connected_grammar_batch_at_rate.argtypes = [vp, vp, u32, u32, u32, u32, vp, u32, u32,
                                                                   C.POINTER(ConnOut)]
        L.sr_fft_mag_batch.argtypes = [vp, vp, u32, u32, vp]
        L.sr_fft_raw_batch.argtypes = [vp, vp, u32, vp]
        L.sr_debug_fft_raw_n.argtypes = [vp, vp, u32, u32, vp]
        L.sr_get_dis_batch.argtypes = [vp, vp, vp, u32, vp]
        L.sr_dtw_limit_batch.argtypes = [vp, vp, vp, vp, vp, u32, vp]
        L.dtw_limit.argtypes = [C.c_uint16, C.c_uint16]
        L.dtw_limit.restype = C.c_uint8
        L.sr_synth_pcm_host.argtypes = [vp, u32, u32, u64, u32]
        L.sr_synth_pcm_dev.argtypes = [vp, u32, u32, u64, u32, vp]
        L.sr_synth_ftr_host.argtypes = [vp, u32, u32, u64, u32, u32]
        L.sr_wav_to_adc12.argtypes = [vp, C.c_size_t, vp, C.c_size_t, vp]
        L.sr_wav_to_adc12.restype = C.c_long
        L.sr_resample_adc12_dev.argtypes = [vp, u32, u32, vp, u32, vp, u32, vp, vp]
        L.noise_atap.argtypes = [vp, C.c_uint16, vp]
        L.noise_atap.restype = None
        L.VAD.argtypes = [vp, C.c_uint16, vp, vp]
        L.VAD.restype = None
        L.get_mfcc.argtypes = [vp, vp, vp]
        L.get_mfcc.restype = None
        L.dtw.argtypes = [vp, vp]
        L.dtw.restype = u32
        L.fft.argtypes = [vp, C.c_uint16]
        L.fft.restype = C.POINTER(C.c_uint32)
        L.get_dis.argtypes = [vp, vp]
        L.get_dis.restype = u32
        _lib = L
    return _lib


def _p(a):
    """void* of a numpy array (must be C-contiguous) or an int device pointer / None."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))


class SrError(RuntimeError):
    pass


class Handle:
    """RAII wrapper of sr_handle. `device` is the CUDA ordinal."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        rc = lib().sr_create(int(device), C.byref(self._h))
        if rc != 0:
            raise SrError("sr_create failed (%d): %s" % (rc, lib().sr_last_error(None).decode()))
        self.n_slot = 0

    def close(self):
        if self._h:
            lib().sr_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise SrError("libspeech_b200 call failed (%d): %s" % (rc, lib().sr_last_error(self._h).decode()))

    # -- plumbing
    def set_stream(self, stream_ptr):
        self._ck(lib().sr_set_stream(self._h, _p(stream_ptr)))

    def use_own_stream(self):
        self._ck(lib().sr_use_own_stream(self._h))

    def sync(self):
        self._ck(lib().sr_sync(self._h))

    def launch_count(self):
        return int(lib().sr_launch_count(self._h))

    def set_transport(self, mode):
        """packed PCM transport of sr_recognise_batch: 0 off, 1 on, -1 automatic"""
        self._ck(lib().sr_set_transport(self._h, int(mode)))

    def transport_stats(self):
        """(packed chunks, plain chunks, bytes copied host -> device) of the last recognise() call on host buffers"""
        a, b, c = C.c_uint32(0), C.c_uint32(0), C.c_uint64(0)
        lib().sr_transport_stats(self._h, C.byref(a), C.byref(b), C.byref(c))
        return int(a.value), int(b.value), int(c.value)

    def unpack12(self, packed, n):
        """device expander of the packed transport alone (test hook): n samples from n/2*3 bytes"""
        packed = np.ascontiguousarray(packed, np.uint8)
        out = np.empty(n, np.uint16)
        self._ck(lib().sr_debug_unpack12(self._h, _p(packed.ctypes.data), n, _p(out.ctypes.data)))
        return out

    def timing_enable(self, max_records):
        self._ck(lib().sr_timing_enable(self._h, max_records))
        self._timing_cap = max_records

    def timing_collect(self):
        """[(tag, ms), ...] for every kernel launched since the last collect (synchronises the stream)"""
        cap = getattr(self, "_timing_cap", 0)
        tags, ms, n = np.zeros(cap, np.uint32), np.zeros(cap, np.float32), C.c_uint32(0)
        self._ck(lib().sr_timing_collect(self._h, _p(tags), _p(ms), cap, C.byref(n)))
        return list(zip(tags[: n.value].tolist(), ms[: n.value].tolist()))

    def set_bank(self, bank, n_slot, slot_stride):
        self._ck(lib().sr_set_bank(self._h, _p(bank), n_slot, slot_stride))
        self.n_slot = n_slot

    def set_bank_dev(self, bank_ptr, n_slot, slot_stride):
        self._ck(lib().sr_set_bank_dev(self._h, _p(bank_ptr), n_slot, slot_stride))
        self.n_slot = n_slot

    # -- host-buffer batched entry points (numpy in / numpy out)
    def noise_atap(self, pcm, n_len, atap=None):
        B, U = pcm.shape
        if atap is None:
            atap = np.zeros(B, ATAP_DTYPE)
        self._ck(lib().sr_noise_atap_batch(self._h, _p(pcm), U, B, n_len, _p(atap)))
        return atap

    def vad(self, pcm, atap, buf_len=None):
        B, U = pcm.shape
        seg = np.zeros((B, 3, 2), np.uint32)
        self._ck(lib().sr_vad_batch(self._h, _p(pcm), U, B, U if buf_len is None else buf_len, _p(atap), _p(seg)))
        return seg

    def mfcc(self, pcm, seg, atap, ftr=None):
        B, U = pcm.shape
        seg = np.ascontiguousarray(seg, np.uint32).reshape(B, -1)
        if ftr is None:
            ftr = np.zeros(B, FTR_DTYPE)
        self._ck(lib().sr_mfcc_batch(self._h, _p(pcm), U, B, _p(seg), seg.shape[1], _p(atap), _p(ftr)))
        return ftr

    def dtw(self, ftr_in, flags=0, band_r=0, want_score=True, want_best=True):
        """every input against the bank (sr_dtw_batch): flags 0 = the greedy walk, DTW_BAND = the banded DP (| DTW_ANY_RATE:
        without the 2:1 length guard), DTW_SYM_P1 = the symmetric P = 1 DP, at radius band_r, each optionally |
        DTW_CHECK_SIGN and | DTW_LIFTER (liftered rows) -> (score [B, n_slot], best_idx [B],
        best_dis [B]), None where not wanted"""
        B = ftr_in.shape[0]
        score = np.zeros((B, self.n_slot), np.uint32) if want_score else None
        bi = np.zeros(B, np.uint32) if want_best else None
        bd = np.zeros(B, np.uint32) if want_best else None
        self._ck(lib().sr_dtw_batch(self._h, _p(ftr_in), B, flags, band_r, _p(score), _p(bi), _p(bd)))
        return score, bi, bd

    def recognise(self, pcm, n_len=2400, want=RECOG_FIELDS, rate=None):
        """spch_recg on captures pcm [B, U] (sr_recognise_batch). rate: None (8 kHz input), or the input rate of
        sr_recognise_batch_at_rate (include/sr_synth.h; any of RESAMPLE_RATES): pcm then counts samples at that rate,
        while n_len and the outputs stay in 8 kHz samples"""
        B, U = pcm.shape
        out = _recog_arrays(B, self.n_slot, want)
        if rate is None:
            self._ck(lib().sr_recognise_batch(self._h, _p(pcm), U, B, n_len, C.byref(_recog_out(out))))
        else:
            self._ck(lib().sr_recognise_batch_at_rate(self._h, _p(pcm), U, B, rate, n_len, C.byref(_recog_out(out))))
        return out

    def enrol(self, pcm, n_len=2400, slot_stride=4096, rate=None):
        """save_mdl on captures pcm [B, U] (sr_enrol_batch): (bank [B, slot_stride] u8, status [B]). rate: None (8 kHz
        input), or the input rate of sr_enrol_batch_at_rate (include/sr_synth.h), as in recognise"""
        B, U = pcm.shape
        bank = np.zeros((B, slot_stride), np.uint8)
        status = np.zeros(B, np.uint8)
        if rate is None:
            self._ck(lib().sr_enrol_batch(self._h, _p(pcm), U, B, n_len, _p(bank), slot_stride, _p(status)))
        else:
            self._ck(lib().sr_enrol_batch_at_rate(self._h, _p(pcm), U, B, rate, n_len, _p(bank), slot_stride, _p(status)))
        return bank, status

    def get_mdl(self, in1, in2, mdl=None):
        n = in1.shape[0]
        if mdl is None:
            mdl = np.zeros(n, FTR_DTYPE)
        dis = np.zeros(n, np.uint32)
        self._ck(lib().sr_get_mdl_batch(self._h, _p(in1), _p(in2), n, _p(mdl), _p(dis)))
        return mdl, dis

    def dtw_path(self, a, b, band_r, with_path=True):
        """banded DP of the pairs (a[p], b[p]) with its optimal warping path (sr_dtw_path_batch): (dis [n], path
        [n, PATH_MAX, 2] of (i, j) points, 0xFF past path_len, path_len [n]); path and path_len are None without with_path"""
        a, b = np.ascontiguousarray(a, FTR_DTYPE), np.ascontiguousarray(b, FTR_DTYPE)
        n = a.shape[0]
        assert b.shape[0] == n
        dis = np.zeros(n, np.uint32)
        path = np.zeros((n, PATH_MAX, 2), np.uint8) if with_path else None
        plen = np.zeros(n, np.uint32) if with_path else None
        self._ck(lib().sr_dtw_path_batch(self._h, _p(a), _p(b), n, int(band_r), _p(path), _p(plen), _p(dis)))
        return dis, path, plen

    def average_bank(self, bank, slot_stride, K, band_r, iters):
        """one template per group of K consecutive slots by DTW barycentre averaging (sr_average_bank): bank [G*K,
        slot_stride] u8 -> (bank_out of the same shape, score [G, K], anchor [G])"""
        bank = np.ascontiguousarray(bank, np.uint8).reshape(-1, slot_stride)
        assert bank.shape[0] % K == 0
        G = bank.shape[0] // K
        out = np.zeros_like(bank)
        score, anchor = np.zeros((G, K), np.uint32), np.zeros(G, np.uint32)
        self._ck(lib().sr_average_bank(self._h, _p(bank), slot_stride, K, G, int(band_r), iters, _p(out), _p(score),
                                       _p(anchor)))
        return out, score, anchor

    def mfcc_long(self, pcm, seg, atap, frm_cap=CONN_FRM_MAX, feat=None):
        """get_mfcc with vv_frm_max replaced by frm_cap (sr_mfcc_long_batch): (feat [B, frm_cap, 12] i16, frm_num [B]);
        rows at or past frm_num keep what `feat` held (zeros when it is None)"""
        B, U = pcm.shape
        seg = np.ascontiguousarray(seg, np.uint32).reshape(B, -1)
        feat = np.zeros((B, frm_cap, 12), np.int16) if feat is None else feat
        assert feat.shape == (B, frm_cap, 12) and feat.dtype == np.int16 and feat.flags["C_CONTIGUOUS"]
        frm = np.zeros(B, np.uint32)
        self._ck(lib().sr_mfcc_long_batch(self._h, _p(pcm), U, B, _p(seg), seg.shape[1], _p(atap), frm_cap, _p(feat), _p(frm)))
        return feat, frm

    def connected(self, feat, frm_num, penalty, max_words, words=None, want_total=True):
        """connected words of feature sequences feat [B, frm_stride, 12] i16 of frm_num [B] frames against the bank
        (sr_connected_batch): (words [B, max_words] WORD_DTYPE, n_words [B], total [B] u64 or None); records past n_words
        keep what `words` held (zeros when it is None)"""
        feat = np.ascontiguousarray(feat, np.int16)
        B, stride = feat.shape[0], feat.shape[1]
        frm_num = np.ascontiguousarray(frm_num, np.uint32)
        words = np.zeros((B, max_words), WORD_DTYPE) if words is None else words
        n_words = np.zeros(B, np.uint32)
        total = np.zeros(B, np.uint64) if want_total else None
        self._ck(lib().sr_connected_batch(self._h, _p(feat), _p(frm_num), stride, B, penalty, max_words, _p(words),
                                          _p(n_words), _p(total)))
        return words, n_words, total

    def recognise_connected(self, pcm, penalty, max_words, n_len=2400, want=CONN_FIELDS, out=None, rate=None):
        """noise_atap -> VAD -> long features of every segment -> connected words (sr_recognise_connected_batch): a dict
        of the sr_conn_out fields named in `want` (or the arrays of `out`, which the call fills in place). rate: None
        (8 kHz input), or the input rate of sr_recognise_connected_batch_at_rate (include/sr_synth.h), as in recognise"""
        B, U = pcm.shape
        if out is None:
            shape = {"atap": (B, ATAP_DTYPE), "seg_off": ((B, 3, 2), np.uint32), "frm_num": ((B, 3), np.uint32),
                     "n_words": (B, np.uint32), "words": ((B, max_words), WORD_DTYPE), "total": (B, np.uint64),
                     "status": (B, np.uint8)}
            out = {k: np.zeros(*shape[k]) for k in CONN_FIELDS if k in want}
        o = ConnOut(*[_p(out.get(k)) for k in CONN_FIELDS])
        if rate is None:
            self._ck(lib().sr_recognise_connected_batch(self._h, _p(pcm), U, B, n_len, penalty, max_words, C.byref(o)))
        else:
            self._ck(lib().sr_recognise_connected_batch_at_rate(self._h, _p(pcm), U, B, rate, n_len, penalty, max_words,
                                                                C.byref(o)))
        return out

    def connected_grammar(self, feat, frm_num, grammar_, penalty, max_words, words=None, want_total=True):
        """connected words under a grammar (sr_connected_grammar_batch), given as (n_states, final_mask, [(from, to,
        cmd_mask), ...]) or a Grammar: (words [B, max_words] WORD_DTYPE, n_words [B], total [B] u64 or None); records
        past n_words keep what `words` held (zeros when it is None)"""
        feat = np.ascontiguousarray(feat, np.int16)
        B, stride = feat.shape[0], feat.shape[1]
        frm_num = np.ascontiguousarray(frm_num, np.uint32)
        words = np.zeros((B, max_words), WORD_DTYPE) if words is None else words
        n_words = np.zeros(B, np.uint32)
        total = np.zeros(B, np.uint64) if want_total else None
        g = grammar(grammar_)
        self._ck(lib().sr_connected_grammar_batch(self._h, _p(feat), _p(frm_num), stride, B, None if g is None else C.byref(g),
                                                  penalty, max_words, _p(words), _p(n_words), _p(total)))
        return words, n_words, total

    def recognise_connected_grammar(self, pcm, grammar_, penalty, max_words, n_len=2400, want=CONN_FIELDS, out=None,
                                    rate=None):
        """noise_atap -> VAD -> long features -> one grammar decode per capture across its segments
        (sr_recognise_connected_grammar_batch): a dict of the sr_conn_out fields named in `want` (or the arrays of `out`,
        filled in place). rate: None (8 kHz input), or the input rate of sr_recognise_connected_grammar_batch_at_rate
        (include/sr_synth.h), as in recognise"""
        B, U = pcm.shape
        if out is None:
            shape = {"atap": (B, ATAP_DTYPE), "seg_off": ((B, 3, 2), np.uint32), "frm_num": ((B, 3), np.uint32),
                     "n_words": (B, np.uint32), "words": ((B, max_words), WORD_DTYPE), "total": (B, np.uint64),
                     "status": (B, np.uint8)}
            out = {k: np.zeros(*shape[k]) for k in CONN_FIELDS if k in want}
        o = ConnOut(*[_p(out.get(k)) for k in CONN_FIELDS])
        g = grammar(grammar_)
        if rate is None:
            self._ck(lib().sr_recognise_connected_grammar_batch(self._h, _p(pcm), U, B, n_len,
                                                                None if g is None else C.byref(g), penalty, max_words,
                                                                C.byref(o)))
        else:
            self._ck(lib().sr_recognise_connected_grammar_batch_at_rate(self._h, _p(pcm), U, B, rate, n_len,
                                                                        None if g is None else C.byref(g), penalty,
                                                                        max_words, C.byref(o)))
        return out

    # -- long-form VAD and per-segment recognition (include/sr_long.h)
    def vad_long_batch(self, pcm, max_segs, n_len=2400, lens=None, atap=None, seg_off=None):
        """long-form noise_atap + VAD of pcm [B, U] (lens [B] samples each, None = U): dict(atap [B], n_segs [B],
        seg_off [B, max_segs, 2]); atap and seg_off are in / out (prefilled bytes stay where nothing is written)"""
        B, U = pcm.shape
        atap = np.zeros(B, ATAP_DTYPE) if atap is None else atap
        seg_off = np.zeros((B, max_segs, 2), np.uint32) if seg_off is None else seg_off
        lens = None if lens is None else np.ascontiguousarray(lens, np.uint32)
        n_segs = np.zeros(B, np.uint32)
        self._ck(lib().sr_vad_long_batch(self._h, _p(pcm), U, B, _p(lens), n_len, max_segs, _p(atap), _p(n_segs),
                                         _p(seg_off) if max_segs else None))
        return dict(atap=atap, n_segs=n_segs, seg_off=seg_off)

    def recognise_long_batch(self, pcm, max_segs, n_len=2400, lens=None, atap=None, segs=None, rate=None):
        """long-form VAD, then spch_recg's decision on every segment: dict(atap [B], n_segs [B], segs [B, max_segs]
        LONG_SEG_DTYPE); atap and segs are in / out. rate: None (8 kHz input, sr_recognise_long_batch), or the input rate
        of sr_recognise_long_batch_at_rate (include/sr_synth.h; any of RESAMPLE_RATES): pcm and lens then count samples
        at that rate, while n_len and the segment offsets stay in 8 kHz samples"""
        B, U = pcm.shape
        atap = np.zeros(B, ATAP_DTYPE) if atap is None else atap
        segs = np.zeros((B, max_segs), LONG_SEG_DTYPE) if segs is None else segs
        lens = None if lens is None else np.ascontiguousarray(lens, np.uint32)
        n_segs = np.zeros(B, np.uint32)
        out = LongOut(_p(atap), _p(n_segs), _p(segs) if max_segs else None)
        if rate is None:
            self._ck(lib().sr_recognise_long_batch(self._h, _p(pcm), U, B, _p(lens), n_len, max_segs, C.byref(out)))
        else:
            self._ck(lib().sr_recognise_long_batch_at_rate(self._h, _p(pcm), U, B, _p(lens), rate, n_len, max_segs,
                                                           C.byref(out)))
        return dict(atap=atap, n_segs=n_segs, segs=segs)

    def vad_long_batch_dev(self, pcm_ptr, U, B, lens_ptr, n_len, max_segs, atap_ptr, n_segs_ptr, seg_ptr):
        self._ck(lib().sr_vad_long_batch_dev(self._h, _p(pcm_ptr), U, B, _p(lens_ptr), n_len, max_segs, _p(atap_ptr),
                                             _p(n_segs_ptr), _p(seg_ptr)))

    def recognise_long_batch_dev(self, pcm_ptr, U, B, lens_ptr, n_len, max_segs, atap_ptr, n_segs_ptr, segs_ptr):
        out = LongOut(_p(atap_ptr), _p(n_segs_ptr), _p(segs_ptr))
        self._ck(lib().sr_recognise_long_batch_dev(self._h, _p(pcm_ptr), U, B, _p(lens_ptr), n_len, max_segs, C.byref(out)))

    # -- one grammar decode per long recording (include/sr_long_grammar.h)
    def connected_grammar_segs(self, feat, seq_seg, seg_frm, grammar_, penalty, max_words, words=None, want_total=True):
        """the grammar decoder over a flat segment table (sr_connected_grammar_segs_batch): feat [rows, 12] i16 (the
        segments' rows back to back), seq_seg [B+1], seg_frm [n_seg] -> (words [B, max_words] WORD_DTYPE, n_words [B],
        total [B] u64 or None); records past n_words keep what `words` held (zeros when it is None)"""
        feat = np.ascontiguousarray(feat, np.int16)
        seq_seg = np.ascontiguousarray(seq_seg, np.uint32)
        seg_frm = np.ascontiguousarray(seg_frm, np.uint32)
        B = len(seq_seg) - 1
        words = np.zeros((B, max_words), WORD_DTYPE) if words is None else words
        n_words = np.zeros(B, np.uint32)
        total = np.zeros(B, np.uint64) if want_total else None
        g = grammar(grammar_)
        self._ck(lib().sr_connected_grammar_segs_batch(self._h, _p(feat) if feat.size else None, _p(seq_seg),
                                                       _p(seg_frm) if seg_frm.size else None, B,
                                                       None if g is None else C.byref(g), penalty, max_words, _p(words),
                                                       _p(n_words), _p(total)))
        return words, n_words, total

    def recognise_long_grammar(self, pcm, grammar_, penalty, max_segs, max_words, n_len=2400, lens=None,
                               want=LONG_GRAM_FIELDS, out=None, rate=None):
        """long-form VAD, long features of every decodable segment and one grammar decode per recording
        (sr_recognise_long_grammar_batch): a dict of the sr_long_gram_out fields named in `want` (or the arrays of `out`,
        filled in place). rate: None (8 kHz input), or the input rate of sr_recognise_long_grammar_batch_at_rate
        (include/sr_synth.h), as in recognise_long_batch"""
        B, U = pcm.shape
        if out is None:
            shape = {"atap": (B, ATAP_DTYPE), "n_segs": (B, np.uint32), "seg_off": ((B, max_segs, 2), np.uint32),
                     "frm_num": ((B, max_segs), np.uint32), "seg_status": ((B, max_segs), np.uint8),
                     "n_words": (B, np.uint32), "words": ((B, max_words), WORD_DTYPE), "total": (B, np.uint64)}
            out = {k: np.zeros(*shape[k]) for k in LONG_GRAM_FIELDS if k in want}
        lens = None if lens is None else np.ascontiguousarray(lens, np.uint32)
        o = LongGramOut(*[_p(out.get(k)) for k in LONG_GRAM_FIELDS])
        g = grammar(grammar_)
        if rate is None:
            self._ck(lib().sr_recognise_long_grammar_batch(self._h, _p(pcm), U, B, _p(lens), n_len,
                                                           None if g is None else C.byref(g), penalty, max_segs, max_words,
                                                           C.byref(o)))
        else:
            self._ck(lib().sr_recognise_long_grammar_batch_at_rate(self._h, _p(pcm), U, B, _p(lens), rate, n_len,
                                                                   None if g is None else C.byref(g), penalty, max_segs,
                                                                   max_words, C.byref(o)))
        return out

    def fft_mag(self, frames):
        n, length = frames.shape
        mag = np.zeros((n, 512), np.uint32)
        self._ck(lib().sr_fft_mag_batch(self._h, _p(frames), length, n, _p(mag)))
        return mag

    def fft_raw(self, packed):
        n = packed.shape[0]
        out = np.zeros((n, 1024), np.uint32)
        self._ck(lib().sr_fft_raw_batch(self._h, _p(packed), n, _p(out)))
        return out

    def fft_raw_n(self, packed, N):
        """the MFCC kernels' shared FFT alone at N = 256 or 1024 (test hook): packed [n, N] -> packed [n, N]"""
        packed = np.ascontiguousarray(packed, np.uint32)
        n = packed.shape[0]
        assert packed.shape == (n, N)
        out = np.zeros((n, N), np.uint32)
        self._ck(lib().sr_debug_fft_raw_n(self._h, _p(packed), N, n, _p(out)))
        return out

    def get_dis(self, a, b):
        n = a.shape[0]
        out = np.zeros(n, np.uint32)
        self._ck(lib().sr_get_dis_batch(self._h, _p(a), _p(b), n, _p(out)))
        return out

    # -- device-pointer entry points (ints / torch data_ptr()), asynchronous on the handle's stream
    def noise_atap_dev(self, pcm_ptr, U, B, n_len, atap_ptr):
        self._ck(lib().sr_noise_atap_batch_dev(self._h, _p(pcm_ptr), U, B, n_len, _p(atap_ptr)))

    def vad_dev(self, pcm_ptr, U, B, buf_len, atap_ptr, seg_ptr):
        self._ck(lib().sr_vad_batch_dev(self._h, _p(pcm_ptr), U, B, buf_len, _p(atap_ptr), _p(seg_ptr)))

    def mfcc_dev(self, pcm_ptr, U, B, seg_ptr, seg_stride, atap_ptr, ftr_ptr):
        self._ck(lib().sr_mfcc_batch_dev(self._h, _p(pcm_ptr), U, B, _p(seg_ptr), seg_stride, _p(atap_ptr), _p(ftr_ptr)))

    def dtw_dev(self, ftr_ptr, B, flags, band_r, score_ptr, bi_ptr, bd_ptr):
        self._ck(lib().sr_dtw_batch_dev(self._h, _p(ftr_ptr), B, flags, band_r, _p(score_ptr), _p(bi_ptr), _p(bd_ptr)))

    # -- the exchange step (NCCL behind the C-ABI)
    def comm_create(self, rank, world, id_bytes):
        buf = (C.c_uint8 * 128).from_buffer_copy(bytes(id_bytes))
        self._ck(lib().sr_comm_create(self._h, rank, world, buf))

    def comm_wait(self):
        self._ck(lib().sr_comm_wait(self._h))

    def allgather_dev(self, send_ptr, recv_ptr, nbytes):
        self._ck(lib().sr_allgather_dev(self._h, _p(send_ptr), _p(recv_ptr), nbytes))

    def recognise_dev_allgather(self, pcm_ptr, U, B, n_len, gathered_score=None, gathered_best=None, **ptrs):
        self._ck(lib().sr_recognise_batch_dev_allgather(self._h, _p(pcm_ptr), U, B, n_len, C.byref(_recog_out(ptrs)),
                                                         _p(gathered_score), _p(gathered_best)))

    def set_dtw_variant(self, v):
        """greedy dtw kernel: 0 static lane = pair, 1 dynamic pair scheduling, -1 library default"""
        self._ck(lib().sr_set_dtw_variant(self._h, int(v)))

    def set_match(self, flags, band_r=0):
        """matcher of the recognition calls: 0 = the reference's greedy walk, DTW_BAND = the banded DP at radius band_r,
        DTW_BAND | DTW_ANY_RATE = the same DP without the 2:1 length guard, DTW_SYM_P1 = the symmetric slope-constrained (P = 1) DP at radius band_r;
        any of them | dtw_knn(k) decides by each command's score e_c, the floor of the mean of its min(k, n_c) smallest
        scores other than DIS_ERR (n_c of them), with the winner's nearest slot as best_idx and e_cmd as best_dis;
        any of them | dtw_reject(q) turns down (ST_REJECT) a decision whose runner-up command is less than q per mille worse
        (under dtw_knn, by the commands' e_c); any of them | DTW_LIFTER scores the liftered rows of inputs and templates"""
        self._ck(lib().sr_set_match(self._h, int(flags), int(band_r)))

    def match(self):
        """(flags, band_r) of the recognition calls' matcher"""
        f, r = C.c_uint32(0), C.c_int(0)
        self._ck(lib().sr_get_match(self._h, C.byref(f), C.byref(r)))
        return int(f.value), int(r.value)

    def set_geometry(self, geom):
        """0 = reference 160/80/1024, 1 = GEOM_B 200/80/256 (extension, parity unpinned)"""
        self._ck(lib().sr_set_geometry(self._h, int(geom)))

    def label(self, cmd):
        """bytes of the command label (commstr, main.c:25-31) or None"""
        p = lib().sr_label(self._h, int(cmd))
        return C.string_at(p) if p else None

    def set_labels(self, labels, stride):
        raw = b"".join(bytes(l)[:stride - 1].ljust(stride, b"\0") for l in labels)
        self._ck(lib().sr_set_labels(self._h, raw, len(labels), stride))

    def recognise_dev(self, pcm_ptr, U, B, n_len, **ptrs):
        self._ck(lib().sr_recognise_batch_dev(self._h, _p(pcm_ptr), U, B, n_len, C.byref(_recog_out(ptrs))))


def comm_unique_id():
    """128 bytes identifying a new communicator (call on one rank, hand to the others)"""
    buf = (C.c_uint8 * 128)()
    rc = lib().sr_comm_unique_id(buf)
    if rc != 0:
        raise SrError("sr_comm_unique_id failed (%d): %s" % (rc, lib().sr_last_error(None).decode()))
    return bytes(buf)


def recognise_multi(handles, pcm, n_len=2400, want=("best_idx", "best_dis", "cmd", "status", "score", "seg_off"),
                    rate=None):
    """sr_recognise_batch_multi: one host call over several handles (one per GPU); numpy in/out. rate: None (8 kHz
    input), or the input rate of sr_recognise_batch_multi_at_rate (include/sr_synth.h), as in Handle.recognise"""
    B, U = pcm.shape
    out = _recog_arrays(B, handles[0].n_slot, want)
    arr = (C.c_void_p * len(handles))(*[h._h for h in handles])
    if rate is None:
        name = "sr_recognise_batch_multi"
        rc = lib().sr_recognise_batch_multi(arr, len(handles), _p(pcm), U, B, n_len, C.byref(_recog_out(out)))
    else:
        name = "sr_recognise_batch_multi_at_rate"
        rc = lib().sr_recognise_batch_multi_at_rate(arr, len(handles), _p(pcm), U, B, rate, n_len, C.byref(_recog_out(out)))
    if rc != 0:
        raise SrError("%s failed (%d): %s" % (name, rc, lib().sr_last_error(None).decode()))
    return out


class StreamPool:
    """sr_stream_pool / sr_stream_group wrapper: chunked capture of S streams, in lock step or ragged
    (include/speech_recog.h, streaming section). `handle` may be a list of handles: the streams are then sharded over
    them (one GPU each).
    rate: None (8 kHz input, sr_streams_create / sr_stream_group_create), or the input rate of sr_streams_create_at_rate /
    sr_stream_group_create_at_rate (include/sr_synth.h; any of RESAMPLE_RATES, 8000 included): chunks then count samples
    at that rate, while max_samples, n_len and event positions stay 8 kHz samples."""

    def __init__(self, handle, n_streams, max_samples, n_len=2400, rate=None):
        self.S, self.L, self.rate = n_streams, max_samples, rate
        self._p = C.c_void_p()
        self.group = isinstance(handle, (list, tuple))
        self.h = handle[0] if self.group else handle
        if self.group:
            arr = (C.c_void_p * len(handle))(*[h._h for h in handle])
            if rate is None:
                rc = lib().sr_stream_group_create(arr, len(handle), n_streams, max_samples, n_len, C.byref(self._p))
            else:
                rc = lib().sr_stream_group_create_at_rate(arr, len(handle), n_streams, max_samples, n_len, rate,
                                                          C.byref(self._p))
            if rc != 0:
                raise SrError("sr_stream_group_create failed (%d): %s" % (rc, lib().sr_last_error(None).decode()))
        elif rate is None:
            handle._ck(lib().sr_streams_create(handle._h, n_streams, max_samples, n_len, C.byref(self._p)))
        else:
            handle._ck(lib().sr_streams_create_at_rate(handle._h, n_streams, max_samples, n_len, rate, C.byref(self._p)))
        self._ev = (StreamEvent * (3 * n_streams))()

    def _ck(self, rc):
        if rc != 0:
            raise SrError("streaming call failed (%d): %s" % (rc, (lib().sr_last_error(None) or b"").decode()))

    def close(self):
        if self._p:
            (lib().sr_stream_group_destroy if self.group else lib().sr_streams_destroy)(self._p)
            self._p = C.c_void_p()

    def reset(self):
        self._ck((lib().sr_stream_group_reset if self.group else lib().sr_streams_reset)(self._p))

    def _events(self, n):
        return [{k: getattr(self._ev[i], k) for k, _ in StreamEvent._fields_} for i in range(n)]

    def push(self, chunk, chunk_len=None, stride=None, max_events=None):
        """chunk: numpy [S, chunk_len] u16 (or a raw host pointer with chunk_len/stride). Returns list of event dicts."""
        if isinstance(chunk, np.ndarray):
            chunk_len, stride, ptr = chunk.shape[1], chunk.strides[0] // 2, chunk.ctypes.data_as(C.c_void_p)
        else:
            ptr = C.c_void_p(int(chunk))
        n = C.c_uint32(0)
        f = lib().sr_stream_group_push if self.group else lib().sr_streams_push
        self._ck(f(self._p, ptr, chunk_len, stride, self._ev, 3 * self.S if max_events is None else max_events, C.byref(n)))
        return self._events(n.value)

    def push_raw(self, ptr, chunk_len, stride, max_events=None):
        """lock-step push from a raw host pointer; returns only the NUMBER of events (they stay in self._ev): what a
        latency measurement should time -- no Python object is built per event"""
        n = C.c_uint32(0)
        f = lib().sr_stream_group_push if self.group else lib().sr_streams_push
        self._ck(f(self._p, C.c_void_p(int(ptr)), chunk_len, stride, self._ev, 3 * self.S if max_events is None else max_events, C.byref(n)))
        return n.value

    def push_ragged(self, chunk, lens, stride=None, max_events=None):
        """chunk: numpy [S, >= max(lens)] u16 (or raw pointer + stride); lens: [S] samples for each stream"""
        lens = np.ascontiguousarray(lens, np.uint32)
        if isinstance(chunk, np.ndarray):
            stride, ptr = chunk.strides[0] // 2, chunk.ctypes.data_as(C.c_void_p)
        else:
            ptr = C.c_void_p(int(chunk))
        n = C.c_uint32(0)
        f = lib().sr_stream_group_push_ragged if self.group else lib().sr_streams_push_ragged
        self._ck(f(self._p, ptr, stride, _p(lens), self._ev, 3 * self.S if max_events is None else max_events, C.byref(n)))
        return self._events(n.value)

    def fetch(self, max_events=None):
        if self.group:
            raise SrError("fetch() is not defined for a stream group: push zero samples to drain its queue")
        n = C.c_uint32(0)
        self._ck(lib().sr_streams_fetch(self._p, self._ev, 3 * self.S if max_events is None else max_events, C.byref(n)))
        return self._events(n.value)

    def pending(self):
        """events queued by a pool's earlier pushes; a group has no such call (its queued events come out with its next
        push, and a push of zero samples drains them)"""
        if self.group:
            raise SrError("pending() is not defined for a stream group: push zero samples to drain its queue")
        return int(lib().sr_streams_pending(self._p))

    def segments(self):
        seg = np.zeros((self.S, 3, 2), np.uint32)
        atap = np.zeros(self.S, ATAP_DTYPE)
        f = lib().sr_stream_group_segments if self.group else lib().sr_streams_segments
        self._ck(f(self._p, _p(seg), _p(atap)))
        return seg, atap


def _row_stride(chunk):
    """row stride of a [S, n] u16 chunk in samples (numpy may report any stride for a dimension of size 1)"""
    assert chunk.dtype == np.uint16
    return chunk.strides[0] // 2 if chunk.shape[0] > 1 else chunk.shape[1]


class LongStreamPool:
    """sr_long_stream_pool wrapper (include/sr_long_stream.h): S live streams of any length, fed in chunks of at most
    max_chunk samples, every segment decided as it closes. atap: [S] ATAP_DTYPE initial values or None (zeros).
    rate: None (8 kHz input, sr_long_streams_create), or the input rate of sr_long_streams_create_at_rate
    (include/sr_synth.h; any of RESAMPLE_RATES, 8000 included): chunks and max_chunk then count samples at that rate,
    while events, n_recv and open_start stay 8 kHz positions."""

    def __init__(self, handle, n_streams, max_chunk, n_len=2400, atap=None, rate=None):
        self.S, self.h, self.rate = n_streams, handle, rate
        self._p = C.c_void_p()
        if rate is None:
            handle._ck(lib().sr_long_streams_create(handle._h, n_streams, max_chunk, n_len, _p(atap), C.byref(self._p)))
        else:
            handle._ck(lib().sr_long_streams_create_at_rate(handle._h, n_streams, max_chunk, n_len, _p(atap), rate,
                                                            C.byref(self._p)))
        self.max_events = int(lib().sr_long_streams_max_events(self._p))
        self._ev = (StreamEvent * self.max_events)()
        self.ring_len = int(lib().sr_long_streams_ring_len(self._p))

    def _ck(self, rc):
        if rc != 0:
            raise SrError("long streaming call failed (%d): %s" % (rc, (lib().sr_last_error(None) or b"").decode()))

    def close(self):
        if self._p:
            lib().sr_long_streams_destroy(self._p)
            self._p = C.c_void_p()

    def reset(self, which=None, atap=None):
        """restart the streams with which[s] != 0 (None: all) from atap[s] (None: zeros)"""
        which = None if which is None else np.ascontiguousarray(which, np.uint8)
        self._ck(lib().sr_long_streams_reset(self._p, _p(which), _p(atap)))

    def _events(self, n, buf=None):
        buf = self._ev if buf is None else buf
        return [{k: getattr(buf[i], k) for k, _ in StreamEvent._fields_} for i in range(n)]

    def _buf(self, max_events):
        if max_events is None or max_events <= self.max_events:
            return self._ev, self.max_events if max_events is None else max_events
        return (StreamEvent * max_events)(), max_events

    def push(self, chunk, chunk_len=None, stride=None, max_events=None, events=None):
        """chunk: numpy [S, chunk_len] u16 (or a raw host pointer with chunk_len / stride). Returns the events as dicts;
        events: a ctypes StreamEvent array to write them to instead (the count is returned)"""
        if isinstance(chunk, np.ndarray):
            chunk_len, stride, ptr = chunk.shape[1], _row_stride(chunk), chunk.ctypes.data_as(C.c_void_p)
        else:
            ptr = C.c_void_p(int(chunk))
        n = C.c_uint32(0)
        buf, m = (events, len(events) if max_events is None else max_events) if events is not None else self._buf(max_events)
        self._ck(lib().sr_long_streams_push(self._p, ptr, chunk_len, stride, buf, m, C.byref(n)))
        return n.value if events is not None else self._events(n.value, buf)

    def push_ragged(self, chunk, lens, stride=None, max_events=None, events=None):
        """chunk: numpy [S, >= max(lens)] u16 (or raw pointer + stride); lens: [S] samples for each stream"""
        lens = np.ascontiguousarray(lens, np.uint32)
        if isinstance(chunk, np.ndarray):
            stride, ptr = _row_stride(chunk), chunk.ctypes.data_as(C.c_void_p)
        else:
            ptr = C.c_void_p(int(chunk))
        n = C.c_uint32(0)
        buf, m = (events, len(events) if max_events is None else max_events) if events is not None else self._buf(max_events)
        self._ck(lib().sr_long_streams_push_ragged(self._p, ptr, stride, _p(lens), buf, m, C.byref(n)))
        return n.value if events is not None else self._events(n.value, buf)

    def fetch(self, max_events=None):
        buf, m = self._buf(max_events)
        n = C.c_uint32(0)
        self._ck(lib().sr_long_streams_fetch(self._p, buf, m, C.byref(n)))
        return self._events(n.value, buf)

    def pending(self):
        return int(lib().sr_long_streams_pending(self._p))

    def state(self):
        """dict(n_recv [S], n_closed [S], open_start [S] (NULL: none open), atap [S])"""
        out = dict(n_recv=np.zeros(self.S, np.uint32), n_closed=np.zeros(self.S, np.uint32),
                   open_start=np.zeros(self.S, np.uint32), atap=np.zeros(self.S, ATAP_DTYPE))
        self._ck(lib().sr_long_streams_state(self._p, _p(out["n_recv"]), _p(out["n_closed"]), _p(out["open_start"]),
                                             _p(out["atap"])))
        return out


def host_alloc_dev(device, nbytes):
    """pinned host memory on `device`'s NUMA node as a numpy uint8 array (keeps the allocation alive through .base)"""
    p = lib().sr_host_alloc_dev(int(device), nbytes)
    if not p:
        raise SrError("sr_host_alloc_dev(%d, %d) failed" % (device, nbytes))
    buf = (C.c_uint8 * nbytes).from_address(p)
    arr = np.frombuffer(buf, np.uint8)
    return arr, p


def host_free(p):
    lib().sr_host_free(C.c_void_p(p))


# ---- synthetic workload (include/sr_synth.h) -------------------------------------------------------
def synth_pcm_host(B, U, seed_base, nwords=1):
    pcm = np.zeros((B, U), np.uint16)
    rc = lib().sr_synth_pcm_host(_p(pcm), U, B, seed_base, nwords)
    if rc != 0:
        raise SrError("sr_synth_pcm_host failed")
    return pcm


def synth_pcm_dev(pcm_ptr, B, U, seed_base, nwords=1, stream_ptr=None):
    rc = lib().sr_synth_pcm_dev(_p(pcm_ptr), U, B, seed_base, nwords, _p(stream_ptr))
    if rc != 0:
        raise SrError("sr_synth_pcm_dev failed")


def synth_ftr_host(B, seed_base, fmin=50, fmax=100, stride=FTR_BYTES):
    buf = np.zeros((B, stride), np.uint8)
    rc = lib().sr_synth_ftr_host(_p(buf), stride, B, seed_base, fmin, fmax)
    if rc != 0:
        raise SrError("sr_synth_ftr_host failed")
    return buf


def wav_to_adc12(wav_bytes, max_samples=1 << 24):
    """(samples u16[n], sample_rate) from the bytes of a RIFF/WAVE PCM file (include/sr_synth.h)"""
    buf = np.frombuffer(wav_bytes, np.uint8).copy()
    out = np.zeros(min(max_samples, max(len(buf), 1)), np.uint16)
    rate = C.c_uint32(0)
    n = lib().sr_wav_to_adc12(_p(buf), len(buf), _p(out), len(out), C.byref(rate))
    if n < 0:
        raise SrError("not a supported PCM WAV file")
    return out[:n].copy(), rate.value


RESAMPLE_RATES = (8000, 11025, 16000, 22050, 32000, 44100, 48000)   # SR_RESAMPLE_RATES
RESAMPLE_U_MAX = 1 << 30       # SR_RESAMPLE_U_MAX: the longest input of resample_adc12_dev


def resample_adc12_dev(in_ptr, U_in, B, lens_ptr, rate, out_ptr, U_out, out_lens_ptr=None, stream_ptr=None):
    """sr_resample_adc12_dev: B recordings of 12-bit codes at `rate` (device [B, U_in], lengths [B] or None) -> device
    [B, U_out] codes at 8 kHz and their lengths [B] (or None), asynchronous on `stream_ptr` (include/sr_synth.h)"""
    rc = lib().sr_resample_adc12_dev(_p(in_ptr), U_in, B, _p(lens_ptr), rate, _p(out_ptr), U_out, _p(out_lens_ptr),
                                     _p(stream_ptr))
    if rc != 0:
        raise SrError("sr_resample_adc12_dev failed (rate %d, U_in %d, B %d, U_out %d)" % (rate, U_in, B, U_out))


def make_bank(ftr, slot_stride=4096, valid=None):
    """Pack feature structs into flash-layout slots (Src/BSP/Flash.H:11-20, Flash.C:41-63): save_sign =
    save_mask, frm_num, rows; the rest of the slot stays erased-flash 0xFF."""
    T = ftr.shape[0]
    bank = np.full((T, slot_stride), 0xFF, np.uint8)
    raw = ftr.view(np.uint8).reshape(T, FTR_BYTES)
    for t in range(T):
        n = int(ftr["frm_num"][t])
        bank[t, 2:4 + 24 * n] = raw[t, 2:4 + 24 * n]
        sign = SAVE_MASK if (valid is None or valid[t]) else 0xFFFF
        bank[t, 0] = sign & 0xFF
        bank[t, 1] = sign >> 8
    return bank


def pack12_host(x, variant=-1):
    """host packer of the packed transport alone (test hook, no GPU): returns (packed bytes, OR of all samples) or None if
    the variant is not available on this CPU"""
    x = np.ascontiguousarray(x, np.uint16)
    dst = np.zeros(x.size // 2 * 3, np.uint8)
    o = lib().sr_debug_pack12_host(int(variant), _p(x.ctypes.data), x.size, _p(dst.ctypes.data))
    return None if o == 0xFFFFFFFF else (dst, int(o))
