"""ctypes binding of the C ABI in include/lyra_b200.h.

``load()`` binds the nvcc-built product library ``lyra_b200/liblyra_b200.so`` and nothing else; it
raises if the library is missing (run ``python -c 'import __graft_entry__ as g; g.build()'``).  There
is no CPU fallback.  (``CApi(path)`` exists so the CPU test tier can bind the test-only emulated
build of the same sources; the package itself never does.)
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
PRODUCT_SO = os.path.join(_HERE, "liblyra_b200.so")
MODEL_DIR = os.path.join(_HERE, "model_coeffs")

OK, EINVAL, ENODEV, EMODEL = 0, -1, -2, -3
HOP = 320
STATS_WORDS = 8
# word indices of one stream's call statistics (lyra_b200_read_stats); 4-6 differ per role
STAT_HOPS, STAT_SAT_OUT, STAT_ENERGY, STAT_LEVEL = 0, 1, 2, 3
STAT_EMPTY, STAT_BITS = 4, 5                       # encoder
STAT_RECEIVED, STAT_CN_HOPS, STAT_EVENTS = 4, 5, 6  # decoder
NUM_FEATURES = 64
MAX_STAGES = 46


class LyraB200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("lyra_b200 error %d: %s" % (code, msg))
        self.code = code


class CApi:
    def __init__(self, so_path):
        if not os.path.exists(so_path):
            raise FileNotFoundError(
                "%s not found: the CUDA extension is not built (python -c 'import __graft_entry__ as g; g.build()')" % so_path)
        L = C.CDLL(so_path)
        vp, ci = C.c_void_p, C.c_int
        sig = {
            "lyra_b200_create": (ci, [C.c_char_p, ci, ci, C.POINTER(vp)]),
            "lyra_b200_create_ex": (ci, [C.c_char_p, ci, ci, ci, C.POINTER(vp)]),
            "lyra_b200_destroy": (None, [vp]),
            "lyra_b200_last_error": (C.c_char_p, [vp]),
            "lyra_b200_max_streams": (ci, [vp]),
            "lyra_b200_tile_streams": (ci, [vp]),
            "lyra_b200_reset": (ci, [vp, vp, ci]),
            "lyra_b200_encode": (ci, [vp, vp, ci, vp, ci, vp]),
            "lyra_b200_decode": (ci, [vp, vp, ci, vp, vp, ci, vp]),
            "lyra_b200_extract_features": (ci, [vp, vp, ci, vp, vp]),
            "lyra_b200_quantize": (ci, [vp, ci, vp, ci, vp, vp]),
            "lyra_b200_dequantize": (ci, [vp, ci, vp, ci, vp]),
            "lyra_b200_generate": (ci, [vp, vp, ci, vp, vp]),
            "lyra_b200_logmel": (ci, [vp, ci, vp, ci, vp, ci, vp]),
            "lyra_b200_set_stream": (ci, [vp, vp]),
            "lyra_b200_encode_device": (ci, [vp, ci, vp, ci, vp]),
            "lyra_b200_decode_device": (ci, [vp, ci, vp, vp, ci, vp]),
            "lyra_b200_synchronize": (ci, [vp]),
            "lyra_b200_noise_update": (ci, [vp, vp, ci, vp, vp, vp, vp]),
            "lyra_b200_decode_track_noise": (ci, [vp, vp, ci, vp, vp, ci, vp, vp]),
            "lyra_b200_decode_track_noise_device": (ci, [vp, ci, vp, vp, ci, vp, vp]),
            "lyra_b200_noise_update_device": (ci, [vp, ci, vp, vp, vp, vp]),
            "lyra_b200_set_split": (ci, [vp, ci]),
            "lyra_b200_set_blocking_sync": (ci, [vp, ci]),
            "lyra_b200_set_graphs": (ci, [vp, ci]),
            "lyra_b200_set_priority": (ci, [vp, ci]),
            "lyra_b200_graph_replays": (C.c_uint64, [vp]),
            "lyra_b200_set_decoder_mode": (ci, [vp, ci]),
            "lyra_b200_decoder_mode": (ci, [vp]),
            "lyra_b200_launch_count": (C.c_uint64, [vp]),
            "lyra_b200_profile_enable": (ci, [vp, ci]),
            "lyra_b200_profile_read": (ci, [vp, vp, vp]),
            "lyra_b200_noise_estimate": (ci, [vp, vp, ci, vp, vp]),
            "lyra_b200_decode_plc": (ci, [vp, vp, ci, vp, vp, ci, vp, vp]),
            "lyra_b200_decode_plc_device": (ci, [vp, ci, vp, vp, ci, vp, vp]),
            "lyra_b200_plc_get_state": (ci, [vp, vp, ci, vp]),
            "lyra_b200_plc_set_state": (ci, [vp, vp, ci, vp]),
            "lyra_b200_cng_generate": (ci, [vp, vp, ci, vp, vp]),
            "lyra_b200_set_cng_seed": (ci, [vp, C.c_uint64]),
            "lyra_b200_encode_dtx": (ci, [vp, vp, ci, vp, ci, vp, vp]),
            "lyra_b200_encode_dtx_device": (ci, [vp, ci, vp, ci, vp, vp]),
            "lyra_b200_set_active_mask": (ci, [vp, vp]),
            "lyra_b200_set_stats": (ci, [vp, ci]),
            "lyra_b200_read_stats": (ci, [vp, ci, vp, ci, vp, ci]),
            "lyra_b200_read_stats_device": (ci, [vp, ci, ci, vp, ci]),
            "lyra_b200_resample": (ci, [vp, ci, vp, ci, ci, vp, ci, vp, ci, vp]),
            "lyra_b200_set_sample_rate": (ci, [vp, ci]),
            "lyra_b200_sample_rate": (ci, [vp]),
            "lyra_b200_set_stream_sample_rates": (ci, [vp, vp, ci, vp]),
            "lyra_b200_stream_sample_rates": (ci, [vp, vp, ci, vp]),
            "lyra_b200_set_stream_bits": (ci, [vp, ci, vp, ci, vp]),
            "lyra_b200_stream_bits": (ci, [vp, ci, vp, ci, vp]),
            "lyra_b200_set_stream_dtx": (ci, [vp, vp, ci, vp]),
            "lyra_b200_stream_dtx": (ci, [vp, vp, ci, vp]),
            "lyra_b200_stream_state_bytes": (ci, [vp]),
            "lyra_b200_export_streams": (ci, [vp, vp, ci, vp]),
            "lyra_b200_import_streams": (ci, [vp, vp, ci, vp]),
            "lyra_b200_copy_streams": (ci, [vp, vp, vp, ci]),
            "lyra_b200_align_streams": (ci, [vp, vp, vp, ci]),
            "lyra_b200_extract_features_device": (ci, [vp, ci, vp, vp]),
            "lyra_b200_quantize_device": (ci, [vp, ci, vp, ci, vp, vp]),
            "lyra_b200_dequantize_device": (ci, [vp, ci, vp, ci, vp]),
            "lyra_b200_generate_device": (ci, [vp, ci, vp, vp]),
            "lyra_b200_logmel_device": (ci, [vp, ci, ci, vp, ci, vp]),
            "lyra_b200_noise_estimate_device": (ci, [vp, ci, vp, vp]),
            "lyra_b200_cng_generate_device": (ci, [vp, ci, vp, vp]),
            "lyra_b200_resample_device": (ci, [vp, ci, ci, ci, vp, ci, vp, ci, vp]),
        }
        for name, (res, args) in sig.items():
            fn = getattr(L, name)   # AttributeError here = the library does not export the declared ABI
            fn.restype = res
            fn.argtypes = args
        self.lib = L
        self.path = so_path

    EXPORTS = ["lyra_b200_create", "lyra_b200_create_ex", "lyra_b200_destroy", "lyra_b200_last_error", "lyra_b200_max_streams",
               "lyra_b200_tile_streams", "lyra_b200_reset", "lyra_b200_encode", "lyra_b200_decode",
               "lyra_b200_extract_features", "lyra_b200_quantize", "lyra_b200_dequantize", "lyra_b200_generate",
               "lyra_b200_logmel", "lyra_b200_set_stream", "lyra_b200_encode_device", "lyra_b200_decode_device",
               "lyra_b200_synchronize", "lyra_b200_noise_update", "lyra_b200_noise_update_device", "lyra_b200_decode_track_noise",
               "lyra_b200_decode_track_noise_device", "lyra_b200_set_split", "lyra_b200_set_blocking_sync", "lyra_b200_set_graphs", "lyra_b200_set_priority", "lyra_b200_graph_replays", "lyra_b200_set_decoder_mode", "lyra_b200_decoder_mode", "lyra_b200_launch_count", "lyra_b200_profile_enable",
               "lyra_b200_profile_read", "lyra_b200_noise_estimate", "lyra_b200_decode_plc", "lyra_b200_decode_plc_device",
               "lyra_b200_plc_get_state", "lyra_b200_plc_set_state", "lyra_b200_cng_generate", "lyra_b200_set_cng_seed",
               "lyra_b200_encode_dtx", "lyra_b200_encode_dtx_device", "lyra_b200_set_active_mask", "lyra_b200_set_stats",
               "lyra_b200_read_stats", "lyra_b200_read_stats_device", "lyra_b200_resample", "lyra_b200_set_sample_rate",
               "lyra_b200_sample_rate", "lyra_b200_set_stream_sample_rates", "lyra_b200_stream_sample_rates", "lyra_b200_set_stream_bits",
               "lyra_b200_stream_bits", "lyra_b200_set_stream_dtx", "lyra_b200_stream_dtx", "lyra_b200_stream_state_bytes", "lyra_b200_export_streams", "lyra_b200_import_streams",
               "lyra_b200_copy_streams", "lyra_b200_align_streams", "lyra_b200_extract_features_device", "lyra_b200_quantize_device",
               "lyra_b200_dequantize_device", "lyra_b200_generate_device", "lyra_b200_logmel_device", "lyra_b200_noise_estimate_device",
               "lyra_b200_cng_generate_device", "lyra_b200_resample_device"]


_product = None


def load():
    """Bind the product library (nvcc build). Fails loudly if it is missing."""
    global _product
    if _product is None:
        _product = CApi(PRODUCT_SO)
    return _product


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _ids(stream_ids, n):
    if stream_ids is None:
        return None
    a = np.ascontiguousarray(stream_ids, dtype=np.int32)
    if a.size != n:
        raise ValueError("stream_ids must have one id per row")
    return a


def _mask(mask, n, what):
    if mask is None:
        return None
    a = np.ascontiguousarray(mask, dtype=np.uint8)
    if a.size != n:
        raise ValueError("%s must have one entry per row" % what)
    return a


def packet_bytes(num_bits):
    return (num_bits + 7) // 8


class Context:
    """One GPU context: weights + the streaming state of ``max_streams`` independent streams (16 kHz unless set_sample_rate)."""

    ROLES = {"both": 3, "encoder": 1, "decoder": 2}

    def __init__(self, max_streams, model_dir=MODEL_DIR, device=0, capi=None, roles="both"):
        self.api = capi or load()
        h = C.c_void_p()
        rc = self.api.lib.lyra_b200_create_ex(str(model_dir).encode(), int(device), int(max_streams), self.ROLES[roles], C.byref(h))
        if rc != OK:
            raise LyraB200Error(rc, (self.api.lib.lyra_b200_last_error(None) or b"").decode())
        self.h = h
        self.max_streams = max_streams

    def close(self):
        if getattr(self, "h", None):
            self.api.lib.lyra_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _check(self, rc):
        if rc != OK:
            raise LyraB200Error(rc, (self.api.lib.lyra_b200_last_error(self.h) or b"").decode())

    @property
    def launch_count(self):
        return int(self.api.lib.lyra_b200_launch_count(self.h))

    @property
    def tile_streams(self):
        return int(self.api.lib.lyra_b200_tile_streams(self.h))

    def reset(self, stream_ids=None, n=None):
        if stream_ids is None:
            n = self.max_streams if n is None else n
            self._check(self.api.lib.lyra_b200_reset(self.h, None, n))
        else:
            a = np.ascontiguousarray(stream_ids, dtype=np.int32)
            self._check(self.api.lib.lyra_b200_reset(self.h, _ptr(a), a.size))

    # ---- moving streams (lyra_b200_export_streams / _import_streams / _copy_streams) ----
    def stream_state_bytes(self):
        return int(self.api.lib.lyra_b200_stream_state_bytes(self.h))

    def export_streams(self, stream_ids=None, n=None):
        """The complete state of the listed streams (default: 0..n-1, n = max_streams) -> uint8[n, stream_state_bytes()]."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        out = np.empty((n, self.stream_state_bytes()), dtype=np.uint8)
        self._check(self.api.lib.lyra_b200_export_streams(self.h, _ptr(ids), n, _ptr(out)))
        return out

    def import_streams(self, records, stream_ids=None):
        """Install exported records into streams `stream_ids` (default: 0..len(records)-1)."""
        recs = np.ascontiguousarray(records, dtype=np.uint8).reshape(-1, self.stream_state_bytes())
        n = recs.shape[0]
        ids = _ids(stream_ids, n)
        self._check(self.api.lib.lyra_b200_import_streams(self.h, _ptr(ids), n, _ptr(recs)))

    def copy_streams(self, src_ids, dst_ids):
        """Stream dst_ids[k] <- the state of stream src_ids[k] (-1: the state at creation); asynchronous on the installed stream."""
        src = np.ascontiguousarray(src_ids, dtype=np.int32).reshape(-1)
        dst = np.ascontiguousarray(dst_ids, dtype=np.int32).reshape(-1)
        if src.size != dst.size:
            raise ValueError("src_ids and dst_ids must have the same length")
        self._check(self.api.lib.lyra_b200_copy_streams(self.h, _ptr(src), _ptr(dst), src.size))

    def align_streams(self, stream_ids, like_ids):
        """Stream stream_ids[k] takes the network hop counters of stream like_ids[k] (-1: those at creation) and computes exactly
        what it computed before; asynchronous on the installed stream."""
        ids = np.ascontiguousarray(stream_ids, dtype=np.int32).reshape(-1)
        like = np.ascontiguousarray(like_ids, dtype=np.int32).reshape(-1)
        if ids.size != like.size:
            raise ValueError("stream_ids and like_ids must have the same length")
        self._check(self.api.lib.lyra_b200_align_streams(self.h, _ptr(ids), _ptr(like), ids.size))

    def set_sample_rate(self, sample_rate_hz):
        """External rate of encode / decode / decode_plc / encode_dtx / decode_track_noise and their *_device twins: 8000, 16000
        (default), 32000 or 48000.  Their PCM rows then hold sample_rate_hz // 50 samples."""
        self._check(self.api.lib.lyra_b200_set_sample_rate(self.h, int(sample_rate_hz)))

    @property
    def sample_rate(self):
        return int(self.api.lib.lyra_b200_sample_rate(self.h))

    def set_stream_sample_rates(self, rates, stream_ids=None):
        """Streams `stream_ids` (default: 0..len(rates)-1) run the fused calls at rates[k] (8000 / 16000 / 32000 / 48000, at most
        sample_rate): they use the first rate // 50 samples of their rows.  Asynchronous on the installed stream."""
        r = np.ascontiguousarray(rates, dtype=np.int32).reshape(-1)
        ids = _ids(stream_ids, r.size)
        self._check(self.api.lib.lyra_b200_set_stream_sample_rates(self.h, _ptr(ids), r.size, _ptr(r)))

    def stream_sample_rates(self, stream_ids=None, n=None):
        """The rate each listed stream runs at (default: streams 0..n-1, n = max_streams) -> int32[n]."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32).reshape(-1)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        out = np.empty(n, dtype=np.int32)
        self._check(self.api.lib.lyra_b200_stream_sample_rates(self.h, _ptr(ids), n, _ptr(out)))
        return out

    def set_stream_bits(self, role, bits, stream_ids=None):
        """Streams `stream_ids` (default: 0..len(bits)-1) of role "encoder" or "decoder" run the fused calls at bits[k] bits per
        packet (a multiple of 4 in 4..184; 0: the call's num_bits, which also sets the packet row size).  Asynchronous on the
        installed stream."""
        b = np.ascontiguousarray(bits, dtype=np.int32).reshape(-1)
        ids = _ids(stream_ids, b.size)
        self._check(self.api.lib.lyra_b200_set_stream_bits(self.h, self.ROLES.get(role, role), _ptr(ids), b.size, _ptr(b)))

    def stream_bits(self, role, stream_ids=None, n=None):
        """The word of each listed stream in `role` (default: streams 0..n-1, n = max_streams) -> int32[n]; 0: the call's."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32).reshape(-1)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        out = np.empty(n, dtype=np.int32)
        self._check(self.api.lib.lyra_b200_stream_bits(self.h, self.ROLES.get(role, role), _ptr(ids), n, _ptr(out)))
        return out

    def set_stream_dtx(self, enable, stream_ids=None):
        """Streams `stream_ids` (default: 0..len(enable)-1) run encode_dtx with DTX on (1, the default) or off (0: every hop is
        encoded, as LyraEncoder with enable_dtx = false).  Encoder role only.  Asynchronous on the installed stream."""
        e = np.ascontiguousarray(enable, dtype=np.int32).reshape(-1)
        ids = _ids(stream_ids, e.size)
        self._check(self.api.lib.lyra_b200_set_stream_dtx(self.h, _ptr(ids), e.size, _ptr(e)))

    def stream_dtx(self, stream_ids=None, n=None):
        """The DTX setting of each listed stream (default: streams 0..n-1, n = max_streams) -> int32[n]; 1: on."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32).reshape(-1)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        out = np.empty(n, dtype=np.int32)
        self._check(self.api.lib.lyra_b200_stream_dtx(self.h, _ptr(ids), n, _ptr(out)))
        return out

    @property
    def hop(self):
        """Samples per PCM row of the codec calls at the context's sample rate."""
        return self.sample_rate // 50

    def encode(self, pcm, num_bits, stream_ids=None):
        pcm = np.ascontiguousarray(pcm, dtype=np.int16).reshape(-1, self.hop)
        n = pcm.shape[0]
        ids = _ids(stream_ids, n)
        out = np.empty((n, packet_bytes(num_bits)), dtype=np.uint8)
        self._check(self.api.lib.lyra_b200_encode(self.h, _ptr(ids), n, _ptr(pcm), num_bits, _ptr(out)))
        return out

    def decode(self, packets, num_bits, stream_ids=None, received=None):
        packets = np.ascontiguousarray(packets, dtype=np.uint8).reshape(-1, packet_bytes(num_bits))
        n = packets.shape[0]
        ids = _ids(stream_ids, n)
        rec = _mask(received, n, "received")
        out = np.empty((n, self.hop), dtype=np.int16)
        self._check(self.api.lib.lyra_b200_decode(self.h, _ptr(ids), n, _ptr(packets), _ptr(rec), num_bits, _ptr(out)))
        return out

    def extract_features(self, pcm, stream_ids=None):
        pcm = np.ascontiguousarray(pcm, dtype=np.int16).reshape(-1, HOP)
        n = pcm.shape[0]
        ids = _ids(stream_ids, n)
        out = np.empty((n, NUM_FEATURES), dtype=np.float32)
        self._check(self.api.lib.lyra_b200_extract_features(self.h, _ptr(ids), n, _ptr(pcm), _ptr(out)))
        return out

    def quantize(self, features, num_bits, want_indices=False):
        f = np.ascontiguousarray(features, dtype=np.float32).reshape(-1, NUM_FEATURES)
        n = f.shape[0]
        out = np.empty((n, packet_bytes(num_bits)), dtype=np.uint8)
        idx = np.empty((n, MAX_STAGES), dtype=np.int32) if want_indices else None
        self._check(self.api.lib.lyra_b200_quantize(self.h, n, _ptr(f), num_bits, _ptr(out), _ptr(idx)))
        return (out, idx) if want_indices else out

    def dequantize(self, packets, num_bits):
        p = np.ascontiguousarray(packets, dtype=np.uint8).reshape(-1, packet_bytes(num_bits))
        out = np.empty((p.shape[0], NUM_FEATURES), dtype=np.float32)
        self._check(self.api.lib.lyra_b200_dequantize(self.h, p.shape[0], _ptr(p), num_bits, _ptr(out)))
        return out

    def generate(self, features, stream_ids=None):
        f = np.ascontiguousarray(features, dtype=np.float32).reshape(-1, NUM_FEATURES)
        n = f.shape[0]
        ids = _ids(stream_ids, n)
        out = np.empty((n, HOP), dtype=np.int16)
        self._check(self.api.lib.lyra_b200_generate(self.h, _ptr(ids), n, _ptr(f), _ptr(out)))
        return out

    def logmel(self, pcm, num_mel_bins=160, bank=0, stream_ids=None):
        pcm = np.ascontiguousarray(pcm, dtype=np.int16).reshape(-1, HOP)
        n = pcm.shape[0]
        ids = _ids(stream_ids, n)
        out = np.empty((n, num_mel_bins), dtype=np.float32)
        self._check(self.api.lib.lyra_b200_logmel(self.h, bank, _ptr(ids), n, _ptr(pcm), num_mel_bins, _ptr(out)))
        return out

    # ---- device-resident variants (raw CUDA device pointers as ints, e.g. torch.Tensor.data_ptr()) ----
    def set_stream(self, cuda_stream_ptr):
        self._check(self.api.lib.lyra_b200_set_stream(self.h, C.c_void_p(cuda_stream_ptr or 0)))

    def set_active_mask(self, mask):
        """Install the active mask of the *_device codec calls: a device pointer (int), a uint8 CUDA tensor (its data_ptr(); the
        caller keeps it alive while calls that read it are queued) or None to uninstall.  Row k = 0: stream k sits the call out."""
        ptr = mask.data_ptr() if hasattr(mask, "data_ptr") else mask
        self._check(self.api.lib.lyra_b200_set_active_mask(self.h, C.c_void_p(ptr or 0)))

    def set_stats(self, enable):
        """Per-stream call statistics of the fused codec calls on (1) or off (0, the default); a host-side setting."""
        self._check(self.api.lib.lyra_b200_set_stats(self.h, 1 if enable else 0))

    def stats(self, role, stream_ids=None, n=None, clear=False):
        """The call statistics of each listed stream in role "encoder" or "decoder" (default: streams 0..n-1, n = max_streams)
        -> uint64[n][STATS_WORDS]; clear zeroes the counters and the energy after reading (the level and event state stay)."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32).reshape(-1)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        out = np.empty((n, STATS_WORDS), dtype=np.uint64)
        self._check(self.api.lib.lyra_b200_read_stats(self.h, self.ROLES.get(role, role), _ptr(ids), n, _ptr(out), 1 if clear else 0))
        return out

    def stats_device(self, role, n, d_out, clear=False):
        """The call statistics of streams 0..n-1 into the device buffer d_out (uint64[n][STATS_WORDS], pointer as int);
        asynchronous on the installed stream."""
        self._check(self.api.lib.lyra_b200_read_stats_device(self.h, self.ROLES.get(role, role), int(n), C.c_void_p(d_out),
                                                             1 if clear else 0))

    def decode_track_noise(self, packets, num_bits, stream_ids=None, received=None):
        """decode() + noise-estimator update of the received streams on the device -> (pcm[n][320], is_noise[n])."""
        packets = np.ascontiguousarray(packets, dtype=np.uint8).reshape(-1, packet_bytes(num_bits))
        n = packets.shape[0]
        ids = _ids(stream_ids, n)
        rec = _mask(received, n, "received")
        out = np.empty((n, self.hop), dtype=np.int16)
        flags = np.empty(n, dtype=np.uint8)
        self._check(self.api.lib.lyra_b200_decode_track_noise(self.h, _ptr(ids), n, _ptr(packets), _ptr(rec), num_bits, _ptr(out), _ptr(flags)))
        return out, flags.astype(bool)

    def decode_track_noise_device(self, n, d_packets, d_received, num_bits, d_pcm, d_is_noise=0):
        self._check(self.api.lib.lyra_b200_decode_track_noise_device(self.h, n, C.c_void_p(d_packets), C.c_void_p(d_received or 0),
                                                                     num_bits, C.c_void_p(d_pcm), C.c_void_p(d_is_noise or 0)))

    def noise_update(self, pcm, stream_ids=None, update_mask=None):
        """NoiseEstimator::ReceiveSamples on one decoded hop per stream -> (is_noise[n] bool, noise_estimate[n][160])."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int16).reshape(-1, HOP)
        n = pcm.shape[0]
        ids = _ids(stream_ids, n)
        mask = _mask(update_mask, n, "update_mask")
        flags = np.empty(n, dtype=np.uint8)
        est = np.empty((n, 160), dtype=np.float32)
        self._check(self.api.lib.lyra_b200_noise_update(self.h, _ptr(ids), n, _ptr(pcm), _ptr(mask), _ptr(flags), _ptr(est)))
        return flags.astype(bool), est

    def noise_estimate(self, n=None, stream_ids=None):
        """Read-only: (noise_estimate[n][160], is_noise[n] bool) of the decoder-side estimators."""
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        est = np.empty((n, 160), dtype=np.float32)
        flags = np.empty(n, dtype=np.uint8)
        self._check(self.api.lib.lyra_b200_noise_estimate(self.h, _ptr(ids), n, _ptr(est), _ptr(flags)))
        return est, flags.astype(bool)

    # ---- packet-loss concealment / comfort noise / DTX ----
    def decode_plc(self, packets, num_bits, stream_ids=None, received=None):
        """One tick of LyraDecoder with the full concealment / comfort-noise / fade behaviour -> (pcm[n][320], is_comfort_noise[n])."""
        packets = np.ascontiguousarray(packets, dtype=np.uint8).reshape(-1, packet_bytes(num_bits))
        n = packets.shape[0]
        ids = _ids(stream_ids, n)
        rec = _mask(received, n, "received")
        out = np.empty((n, self.hop), dtype=np.int16)
        cn = np.empty(n, dtype=np.uint8)
        self._check(self.api.lib.lyra_b200_decode_plc(self.h, _ptr(ids), n, _ptr(packets), _ptr(rec), num_bits, _ptr(out), _ptr(cn)))
        return out, cn.astype(bool)

    def decode_plc_device(self, n, d_packets, d_received, num_bits, d_pcm, d_is_cn=0):
        self._check(self.api.lib.lyra_b200_decode_plc_device(self.h, n, C.c_void_p(d_packets), C.c_void_p(d_received or 0), num_bits,
                                                             C.c_void_p(d_pcm), C.c_void_p(d_is_cn or 0)))

    def plc_state(self, n=None, stream_ids=None):
        ids = None if stream_ids is None else np.ascontiguousarray(stream_ids, dtype=np.int32)
        n = ids.size if ids is not None else (self.max_streams if n is None else n)
        st = np.empty((n, 3), dtype=np.int32)
        self._check(self.api.lib.lyra_b200_plc_get_state(self.h, _ptr(ids), n, _ptr(st)))
        return st

    def set_plc_state(self, state, stream_ids=None):
        st = np.ascontiguousarray(state, dtype=np.int32).reshape(-1, 3)
        ids = _ids(stream_ids, st.shape[0])
        self._check(self.api.lib.lyra_b200_plc_set_state(self.h, _ptr(ids), st.shape[0], _ptr(st)))

    def cng_generate(self, features, stream_ids=None):
        f = np.ascontiguousarray(features, dtype=np.float32).reshape(-1, 160)
        n = f.shape[0]
        ids = _ids(stream_ids, n)
        out = np.empty((n, HOP), dtype=np.int16)
        self._check(self.api.lib.lyra_b200_cng_generate(self.h, _ptr(ids), n, _ptr(f), _ptr(out)))
        return out

    def set_cng_seed(self, seed):
        self._check(self.api.lib.lyra_b200_set_cng_seed(self.h, int(seed)))

    def encode_dtx(self, pcm, num_bits, stream_ids=None):
        """LyraEncoder::Encode with DTX -> (packets[n][P], packet_bytes[n]: P, or 0 for an empty (noise) packet)."""
        pcm = np.ascontiguousarray(pcm, dtype=np.int16).reshape(-1, self.hop)
        n = pcm.shape[0]
        ids = _ids(stream_ids, n)
        out = np.empty((n, packet_bytes(num_bits)), dtype=np.uint8)
        sizes = np.empty(n, dtype=np.int32)
        self._check(self.api.lib.lyra_b200_encode_dtx(self.h, _ptr(ids), n, _ptr(pcm), num_bits, _ptr(out), _ptr(sizes)))
        return out, sizes

    def encode_dtx_device(self, n, d_pcm, num_bits, d_packets, d_is_noise):
        self._check(self.api.lib.lyra_b200_encode_dtx_device(self.h, n, C.c_void_p(d_pcm), num_bits, C.c_void_p(d_packets), C.c_void_p(d_is_noise)))

    def resample(self, audio, external_rate_hz, to_internal, stream_ids=None):
        """Resampler::Resample for n streams -> list of int16 arrays (one per stream; lengths may differ by one when down-sampling)."""
        a = np.ascontiguousarray(audio, dtype=np.int16)
        a = a.reshape(1, -1) if a.ndim == 1 else a
        n, n_in = a.shape
        ids = _ids(stream_ids, n)
        ratio = (16000 / external_rate_hz) if to_internal else (external_rate_hz / 16000)
        stride = int(np.ceil(n_in * ratio)) + 1
        out = np.zeros((n, stride), dtype=np.int16)
        counts = np.zeros(n, dtype=np.int32)
        self._check(self.api.lib.lyra_b200_resample(self.h, 1 if to_internal else 0, _ptr(ids), n, int(external_rate_hz), _ptr(a), n_in,
                                                    _ptr(out), stride, _ptr(counts)))
        return [out[k, :counts[k]].copy() for k in range(n)]

    def noise_update_device(self, n, d_pcm, d_mask, d_is_noise, d_estimate):
        self._check(self.api.lib.lyra_b200_noise_update_device(self.h, n, C.c_void_p(d_pcm), C.c_void_p(d_mask or 0),
                                                               C.c_void_p(d_is_noise or 0), C.c_void_p(d_estimate or 0)))

    def encode_device(self, n, d_pcm, num_bits, d_packets):
        self._check(self.api.lib.lyra_b200_encode_device(self.h, n, C.c_void_p(d_pcm), num_bits, C.c_void_p(d_packets)))

    def decode_device(self, n, d_packets, d_received, num_bits, d_pcm):
        self._check(self.api.lib.lyra_b200_decode_device(self.h, n, C.c_void_p(d_packets), C.c_void_p(d_received or 0),
                                                         num_bits, C.c_void_p(d_pcm)))

    # the plugin-level calls on device buffers (streams 0..n-1, asynchronous on the installed stream; pointers as ints)
    def extract_features_device(self, n, d_pcm, d_features):
        self._check(self.api.lib.lyra_b200_extract_features_device(self.h, n, C.c_void_p(d_pcm), C.c_void_p(d_features)))

    def quantize_device(self, n, d_features, num_bits, d_packets, d_indices=0):
        self._check(self.api.lib.lyra_b200_quantize_device(self.h, n, C.c_void_p(d_features), num_bits, C.c_void_p(d_packets),
                                                           C.c_void_p(d_indices or 0)))

    def dequantize_device(self, n, d_packets, num_bits, d_features):
        self._check(self.api.lib.lyra_b200_dequantize_device(self.h, n, C.c_void_p(d_packets), num_bits, C.c_void_p(d_features)))

    def generate_device(self, n, d_features, d_pcm):
        self._check(self.api.lib.lyra_b200_generate_device(self.h, n, C.c_void_p(d_features), C.c_void_p(d_pcm)))

    def logmel_device(self, n, d_pcm, d_out, num_mel_bins=160, bank=0):
        self._check(self.api.lib.lyra_b200_logmel_device(self.h, bank, n, C.c_void_p(d_pcm), num_mel_bins, C.c_void_p(d_out)))

    def noise_estimate_device(self, n, d_estimate, d_is_noise):
        self._check(self.api.lib.lyra_b200_noise_estimate_device(self.h, n, C.c_void_p(d_estimate or 0), C.c_void_p(d_is_noise or 0)))

    def cng_generate_device(self, n, d_features, d_pcm):
        self._check(self.api.lib.lyra_b200_cng_generate_device(self.h, n, C.c_void_p(d_features), C.c_void_p(d_pcm)))

    def resample_device(self, n, external_rate_hz, to_internal, d_in, in_samples, d_out, out_stride, d_counts=0):
        """Rows of in_samples -> rows of out_stride samples; the first d_counts[k] of row k are written (d_counts may be 0)."""
        self._check(self.api.lib.lyra_b200_resample_device(self.h, 1 if to_internal else 0, n, int(external_rate_hz), C.c_void_p(d_in),
                                                           in_samples, C.c_void_p(d_out), out_stride, C.c_void_p(d_counts or 0)))

    def synchronize(self):
        self._check(self.api.lib.lyra_b200_synchronize(self.h))

    def set_decoder_mode(self, mode):
        """mode: "exact" (bit-identical PCM, default) or "tensor" (split-precision TF32 tensor-core decoder)."""
        self._check(self.api.lib.lyra_b200_set_decoder_mode(self.h, {"exact": 0, "tensor": 1}[mode]))

    def set_blocking_sync(self, enable):
        self._check(self.api.lib.lyra_b200_set_blocking_sync(self.h, 1 if enable else 0))

    def set_graphs(self, enable):
        self._check(self.api.lib.lyra_b200_set_graphs(self.h, 1 if enable else 0))

    def set_priority(self, priority):
        self._check(self.api.lib.lyra_b200_set_priority(self.h, int(priority)))

    def graph_replays(self):
        return int(self.api.lib.lyra_b200_graph_replays(self.h))

    def set_split(self, parts):
        self._check(self.api.lib.lyra_b200_set_split(self.h, int(parts)))

    KERNEL_NAMES = ["EncoderKernelA", "EncoderKernelB", "RvqEncodeKernel", "RvqDecodeKernel", "DecoderKernelC",
                    "DecoderKernelD", "LogMelKernel", "NoiseEstimatorKernel"]

    def profile_enable(self, enable=True):
        self._check(self.api.lib.lyra_b200_profile_enable(self.h, 1 if enable else 0))

    def profile_read(self):
        """-> {kernel name: (total ms, launches)} since profiling was enabled (CUDA events on the launch stream)."""
        ms = (C.c_double * len(self.KERNEL_NAMES))()
        cnt = (C.c_uint64 * len(self.KERNEL_NAMES))()
        self._check(self.api.lib.lyra_b200_profile_read(self.h, ms, cnt))
        return {k: (ms[i], int(cnt[i])) for i, k in enumerate(self.KERNEL_NAMES)}
