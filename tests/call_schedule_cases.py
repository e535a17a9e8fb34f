"""Cases for the launch schedule and the argument checks of the ten fused codec calls (encode, encode_dtx, decode,
decode_track_noise, decode_plc and their *_device twins), shared by the CPU tier (emulated kernels) and the GPU tier.

A call adds a fixed number of launches to lyra_b200_launch_count (what bench.py reports as gpu_launches).  With P sub-batches
and R = 1 when the context converts (a rate other than 16 kHz, or some stream with a rate of its own), else 0:
    encode, decode                  P * (3 + R)
    encode_dtx, decode_track_noise  P * (5 + R)
    decode_plc                      1 + P * (7 + R)
A refused call returns EINVAL and launches nothing.  The calls go through the raw C functions, so NULL pointers can be passed."""
import numpy as np

EINVAL = -1
MAX_ROW = 960                # PCM samples per row at 48 kHz: the buffers fit every rate
MAX_PACKET = 23              # bytes of a 184-bit packet

# call -> (C function, arguments); every pointer argument is named after the buffer it takes
SIGNATURES = {
    "encode": ("lyra_b200_encode", ("ctx", "ids", "n", "pcm", "bits", "packets")),
    "encode_dtx": ("lyra_b200_encode_dtx", ("ctx", "ids", "n", "pcm", "bits", "packets", "sizes")),
    "decode": ("lyra_b200_decode", ("ctx", "ids", "n", "packets", "received", "bits", "out")),
    "decode_track_noise": ("lyra_b200_decode_track_noise", ("ctx", "ids", "n", "packets", "received", "bits", "out", "flags")),
    "decode_plc": ("lyra_b200_decode_plc", ("ctx", "ids", "n", "packets", "received", "bits", "out", "flags")),
    "encode_device": ("lyra_b200_encode_device", ("ctx", "n", "pcm", "bits", "packets")),
    "encode_dtx_device": ("lyra_b200_encode_dtx_device", ("ctx", "n", "pcm", "bits", "packets", "flags")),
    "decode_device": ("lyra_b200_decode_device", ("ctx", "n", "packets", "received", "bits", "out")),
    "decode_track_noise_device": ("lyra_b200_decode_track_noise_device", ("ctx", "n", "packets", "received", "bits", "out", "flags")),
    "decode_plc_device": ("lyra_b200_decode_plc_device", ("ctx", "n", "packets", "received", "bits", "out", "flags")),
}
# the pointers each call refuses when NULL; its other pointers are optional
REQUIRED = {
    "encode": ("pcm", "packets"), "encode_dtx": ("pcm", "packets", "sizes"), "decode": ("packets", "out"),
    "decode_track_noise": ("packets", "out"), "decode_plc": ("packets", "out"),
    "encode_device": ("pcm", "packets"), "encode_dtx_device": ("pcm", "packets", "flags"), "decode_device": ("packets", "out"),
    "decode_track_noise_device": ("packets", "out"), "decode_plc_device": ("packets", "out"),
}
PER_PART = {"encode": 3, "encode_dtx": 5, "decode": 3, "decode_track_noise": 5, "decode_plc": 7}
SETTINGS = ("16k", "48k", "8k_stream_in_16k")


def base(call):
    return call[:-len("_device")] if call.endswith("_device") else call


def expected_launches(call, parts, converts):
    c = base(call)
    return (1 if c == "decode_plc" else 0) + parts * (PER_PART[c] + (1 if converts else 0))


class Buffers:
    """Host buffers (numpy) and device buffers (mem: parity_cases.HostMem or test_gpu_parity.TorchMem) of `rows` rows for every
    pointer a call takes; pointers(device) -> {name: address}"""

    def __init__(self, mem, rows, seed=0):
        rng = np.random.default_rng(seed)
        pcm = rng.integers(-8192, 8192, size=(rows, MAX_ROW), dtype=np.int16)
        packets = rng.integers(0, 256, size=(rows, MAX_PACKET), dtype=np.uint8)
        received = (rng.random(rows) >= 0.3).astype(np.uint8)
        self.host = dict(pcm=pcm, packets=packets, received=received, out=np.zeros((rows, MAX_ROW), np.int16),
                         flags=np.zeros(rows, np.uint8), sizes=np.zeros(rows, np.int32))
        self.mem = mem
        self.dev = {}
        for name, a in self.host.items():
            if name == "sizes":
                continue                      # packet_bytes is a host array in both encode_dtx calls
            self.dev[name] = mem.zeros(a.shape, a.dtype)
            mem.put(self.dev[name], a)

    def pointers(self, device):
        ptrs = {k: a.ctypes.data for k, a in self.host.items()}
        if device:
            ptrs.update({k: self.mem.ptr(t) for k, t in self.dev.items()})
        return ptrs


def raw_call(c, call, bufs, n, bits, ids=None, **override):
    """`call` on context c through c.api.lib with bufs' pointers; override: argument name -> value (None: NULL) -> the return code"""
    fn, params = SIGNATURES[call]
    ptrs = bufs.pointers(call.endswith("_device"))
    ids_arr = None if ids is None else np.ascontiguousarray(ids, dtype=np.int32)
    values = dict(ptrs, ctx=c.h, n=n, bits=bits, ids=None if ids_arr is None else ids_arr.ctypes.data)
    values.update(override)
    return getattr(c.api.lib, fn)(*[values[p] for p in params])


def make_context(Context, api, mem, max_streams, setting, roles="both"):
    c = Context(max_streams, capi=api, roles=roles)
    if mem.stream is not None:
        c.set_stream(mem.stream)
    if setting == "48k":
        c.set_sample_rate(48000)
    elif setting == "8k_stream_in_16k":
        c.set_stream_sample_rates([8000], [1])       # one stream at a rate of its own: the context converts at 16 kHz
    else:
        assert setting == "16k", setting
    return c


def run_launch_counts(Context, api, mem, *, setting, max_streams, n, sparse_ids=None, modes=("exact", "tensor"), splits=(None,),
                      bits=64):
    """Every fused call's launch count in one context at `setting`, in each decoder mode and split: dense calls over streams
    0..n-1 with every pointer given and with every optional pointer NULL, and host-buffer calls over sparse_ids.  splits:
    None keeps the default split, which must leave n in one sub-batch (P = 1); a number sets it and is P (n must be large
    enough for that many sub-batches)."""
    converts = setting != "16k"
    c = make_context(Context, api, mem, max_streams, setting)
    bufs = Buffers(mem, max_streams)
    optional = {call: [p for p in params if p not in REQUIRED[call] and p not in ("ctx", "ids", "n", "bits")]
                for call, (_, params) in SIGNATURES.items()}
    for mode in modes:
        c.set_decoder_mode(mode)
        for split in splits:
            if split is not None:
                c.set_split(split)
            parts = 1 if split is None else split
            for call in SIGNATURES:
                for nulls in ([], optional[call]) if optional[call] else ([],):
                    l0 = c.launch_count
                    rc = raw_call(c, call, bufs, n, bits, **{p: None for p in nulls})
                    assert rc == 0, "%s (%s, %s mode, NULL %s) failed: %d" % (call, setting, mode, nulls, rc)
                    got, want = c.launch_count - l0, expected_launches(call, parts, converts)
                    assert got == want, "%s (%s, %s mode, split %s, n %d, NULL %s): %d launches, expected %d" % (
                        call, setting, mode, split, n, nulls, got, want)
            if sparse_ids is None:
                continue
            for call in PER_PART:
                l0 = c.launch_count
                rc = raw_call(c, call, bufs, len(sparse_ids), bits, ids=sparse_ids)
                assert rc == 0, "%s (%s, %s mode, sparse) failed: %d" % (call, setting, mode, rc)
                got, want = c.launch_count - l0, expected_launches(call, 1, converts)
                assert got == want, "%s (%s, %s mode, sparse ids %s): %d launches, expected %d" % (
                    call, setting, mode, list(sparse_ids), got, want)
    c.close()


def run_rejections(Context, api, mem, *, max_streams=16, n=4, bits=64):
    """Each call refuses, with EINVAL and no launch: a context without the call's role, 0 / 62 / 185 bits, n = 0, n > max_streams,
    a NULL context, each pointer it requires as NULL, and (host-buffer calls) an id out of range or repeated.  The same calls with
    valid arguments succeed."""
    full = make_context(Context, api, mem, max_streams, "16k")
    encoder_only = make_context(Context, api, mem, max_streams, "16k", roles="encoder")
    decoder_only = make_context(Context, api, mem, max_streams, "16k", roles="decoder")
    bufs = Buffers(mem, max_streams + 1)

    def refused(c, call, what, **kw):
        kw.setdefault("n", n)
        kw.setdefault("bits", bits)
        l0 = c.launch_count
        rc = raw_call(c, call, bufs, **kw)
        assert rc == EINVAL, "%s accepted %s: %d" % (call, what, rc)
        assert c.launch_count == l0, "%s launched %d kernels for %s" % (call, c.launch_count - l0, what)

    for call, (_, params) in SIGNATURES.items():
        own = encoder_only if call.startswith("encode") else decoder_only
        other = decoder_only if call.startswith("encode") else encoder_only
        for ctx in (full, own):
            assert raw_call(ctx, call, bufs, n, bits) == 0, call
        refused(other, call, "a context without its role")
        for b in (0, 62, 185):
            refused(full, call, "%d bits" % b, bits=b)
        for m in (0, max_streams + 1):
            refused(full, call, "n = %d" % m, n=m)
        refused(full, call, "a NULL context", ctx=None)
        for p in REQUIRED[call]:
            refused(full, call, "a NULL %s" % p, **{p: None})
        if "ids" in params:
            refused(full, call, "an id out of range", ids=[0, 1, 2, max_streams])
            refused(full, call, "a repeated id", ids=[0, 3, 5, 3])
    for c in (full, encoder_only, decoder_only):
        c.close()
