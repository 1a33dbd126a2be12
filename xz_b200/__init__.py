"""xz_b200 -- H100-native LZMA2 / .xz block path behind liblzma's API surface.

The product is the C-ABI library ``libxzb200.so`` (hand-written sm_90a CUDA + C++ host code,
see ``include/xzb200.h``); this module is a thin ctypes mirror of it, named after the
liblzma calls it stands in for, so that tests and ``bench.py`` read like callers of the
reference.  There is no CPU fallback: importing works anywhere, but creating a
:class:`Context` without the built library or without a CUDA device raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libxzb200.so")

LZMA_OK, LZMA_STREAM_END, LZMA_UNSUPPORTED_CHECK, LZMA_MEM_ERROR = 0, 1, 3, 5
LZMA_FORMAT_ERROR, LZMA_OPTIONS_ERROR, LZMA_DATA_ERROR, LZMA_BUF_ERROR, LZMA_PROG_ERROR = 7, 8, 9, 10, 11
LZMA_CHECK_NONE, LZMA_CHECK_CRC32, LZMA_CHECK_CRC64 = 0, 1, 4
LZMA_PRESET_EXTREME = 0x80000000
LZMA_MF_HC3, LZMA_MF_HC4, LZMA_MF_BT2, LZMA_MF_BT3, LZMA_MF_BT4 = 0x03, 0x04, 0x12, 0x13, 0x14
LZMA_MODE_FAST, LZMA_MODE_NORMAL = 1, 2


class LzmaOptions(C.Structure):
    """xzb_lzma_options == the fields of lzma_options_lzma the LZMA2 encoder reads."""
    _fields_ = [(n, C.c_uint32) for n in ("dict_size", "lc", "lp", "pb", "mode", "nice_len", "mf", "depth")]


class IndexRecord(C.Structure):
    _fields_ = [("unpadded_size", C.c_uint64), ("uncompressed_size", C.c_uint64)]


class Stats(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("ms_total", "ms_h2d", "ms_d2h", "ms_mf_prep", "ms_mf", "ms_parse", "ms_other", "ms_decode")] + \
               [(n, C.c_uint64) for n in ("gpu_launches", "n_blocks", "n_positions", "n_symbols", "n_chunks_lzma", "n_chunks_raw",
                                          "n_fallback_blocks", "mf_bytes_algorithmic")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class BlockDecoderStats(C.Structure):
    """xzb_block_decoder_counters: pieces, bytes, window slides, device times of one resumable Block decoder."""
    _fields_ = [(n, C.c_uint64) for n in ("pieces", "in_bytes", "out_bytes", "slides", "bytes_slid", "window_bytes", "max_history")] + \
               [(n, C.c_double) for n in ("ms_decode", "ms_check", "ms_d2h")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class XzError(RuntimeError):
    def __init__(self, code, msg=""):
        super().__init__(f"lzma_ret {code}: {msg}")
        self.code = code


_lib = None


def lib():
    """Load libxzb200.so; fails loudly when the CUDA extension has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f"{LIB_PATH} is missing: build it with __graft_entry__.build() (nvcc, sm_90a). "
                               "xz_b200 has no CPU fallback.")
        L = C.CDLL(LIB_PATH)
        L.xzb_block_bound.restype = C.c_uint64
        L.xzb_block_bound.argtypes = [C.c_uint64]
        L.xzb_stream_bound.restype = C.c_uint64
        L.xzb_stream_bound.argtypes = [C.c_uint64, C.c_uint64]
        L.xzb_index_encode.restype = C.c_uint64
        L.xzb_last_error.restype = C.c_char_p
        L.xzb_ctx_create.argtypes = [C.POINTER(C.c_void_p), C.c_int]
        L.xzb_ctx_destroy.argtypes = [C.c_void_p]
        L.xzb_get_stats.argtypes = [C.c_void_p, C.POINTER(Stats)]
        L.xzb_last_error.argtypes = [C.c_void_p]
        L.xzb_encode_blocks_device.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(LzmaOptions), C.c_uint32, C.c_uint64,
                                               C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(IndexRecord)]
        L.xzb_encode_blocks_host.argtypes = L.xzb_encode_blocks_device.argtypes
        L.xzb_stream_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(LzmaOptions), C.c_uint32, C.c_uint64,
                                        C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
        L.xzb_stream_buffer_bound.argtypes = [C.c_uint64]
        L.xzb_stream_buffer_bound.restype = C.c_uint64
        L.xzb_stream_buffer_encode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(LzmaOptions), C.c_uint32,
                                               C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
        L.xzb_stream_buffer_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64),
                                               C.POINTER(C.c_uint64), C.c_uint32]
        L.xzb_stream_decode_flags.argtypes = L.xzb_stream_buffer_decode.argtypes
        P64, P32 = C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)
        L.xzb_stream_buffer_encode_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, P64, P64, C.POINTER(LzmaOptions), C.c_uint32,
                                                     C.c_void_p, P64, P64, P64, P32]
        L.xzb_stream_buffer_encode_batch_device.argtypes = L.xzb_stream_buffer_encode_batch.argtypes
        L.xzb_stream_encode_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, P64, P64, C.POINTER(LzmaOptions), C.c_uint32, C.c_uint64,
                                              C.c_void_p, P64, P64, P64, P32]
        L.xzb_stream_encode_batch_device.argtypes = L.xzb_stream_encode_batch.argtypes
        L.xzb_stream_buffer_decode_batch.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, P64, P64, C.c_void_p, P64, P64, P64, P64, P32,
                                                     C.c_uint32]
        L.xzb_stream_buffer_decode_batch_device.argtypes = L.xzb_stream_buffer_decode_batch.argtypes
        L.xzb_stream_decode.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]
        L.xzb_decode_blocks_device.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64),
                                               C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.c_uint32, C.c_uint32, C.c_void_p,
                                               C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)]
        L.xzb_device_alloc.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint64]
        L.xzb_device_free.argtypes = [C.c_void_p, C.c_void_p]
        L.xzb_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        L.xzb_memcpy_d2h.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64]
        L.xzb_block_decoder_create.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
        L.xzb_block_decoder_code.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, P64, C.c_void_p, C.c_uint64, P64, C.c_uint32]
        L.xzb_block_decoder_record.argtypes = [C.c_void_p, C.POINTER(IndexRecord)]
        L.xzb_block_decoder_stats.argtypes = [C.c_void_p, C.POINTER(BlockDecoderStats)]
        L.xzb_block_decoder_destroy.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def lzma_lzma_preset(preset):
    """lzma_lzma_preset(): LZMA2 options of an xz preset level (optionally | LZMA_PRESET_EXTREME)."""
    o = LzmaOptions()
    if lib().xzb_lzma_preset(C.byref(o), C.c_uint32(preset)) != 0:
        raise XzError(LZMA_OPTIONS_ERROR, f"bad preset {preset:#x}")
    return o


def lzma_block_buffer_bound(n):
    return lib().xzb_block_bound(n)


def stream_bound(n, block_size):
    return lib().xzb_stream_bound(n, block_size)


def _ptr(buf):
    """(address, keepalive) of a bytes / bytearray / ctypes array / object with data_ptr() or an int address."""
    if isinstance(buf, int):
        return buf, None
    if hasattr(buf, "data_ptr"):
        return buf.data_ptr(), buf
    if isinstance(buf, (bytes, bytearray)):
        a = (C.c_char * len(buf)).from_buffer_copy(buf) if isinstance(buf, bytes) else (C.c_char * len(buf)).from_buffer(buf)
        return C.addressof(a), a
    return C.addressof(buf), buf


class Context:
    """One per process / GPU: the stand-in for liblzma's worker-thread pool (xzb_ctx)."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        r = lib().xzb_ctx_create(C.byref(self._h), device)
        if r != LZMA_OK:
            raise XzError(r, "xzb_ctx_create failed: no usable CUDA device (no CPU fallback exists)")

    def close(self):
        if self._h:
            lib().xzb_ctx_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self):
        return (lib().xzb_last_error(self._h) or b"").decode()

    def stats(self):
        s = Stats()
        lib().xzb_get_stats(self._h, C.byref(s))
        return s

    def set_filters(self, filters=()):
        """Filters in front of LZMA2 for the following encode calls: [(id, arg), ...] with the XZB_FILTER_ID_* of
        include/xzb200.h (arg = Delta distance or BCJ start offset); () = LZMA2 alone."""
        arr = (C.c_uint32 * (2 * max(1, len(filters))))()
        for i, (fid, arg) in enumerate(filters):
            arr[2 * i] = fid; arr[2 * i + 1] = arg
        r = lib().xzb_ctx_set_filters(self._h, arr, C.c_uint32(len(filters)))
        if r != LZMA_OK:
            raise XzError(r, self._err())

    # ---- lzma_stream_encoder_mt + lzma_code(FINISH) on host buffers ----
    def stream_encode_into(self, src, n, opts, check, block_size, dst, cap):
        sp, _k1 = _ptr(src)
        dp, _k2 = _ptr(dst)
        sz = C.c_uint64()
        r = lib().xzb_stream_encode(self._h, sp, n, C.byref(opts), check, block_size, dp, cap, C.byref(sz))
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return sz.value

    def stream_encode(self, data, preset=6, block_size=0, check=LZMA_CHECK_CRC64, opts=None, n=None):
        o = opts if opts is not None else lzma_lzma_preset(preset)
        n = len(data) if n is None else n
        bs = block_size if block_size else max(3 * o.dict_size, 1 << 20)
        cap = stream_bound(n, bs)
        out = (C.c_uint8 * cap)()
        size = self.stream_encode_into(data, n, o, check, block_size, out, cap)
        return bytes(out[:size])

    # ---- lzma_stream_buffer_encode / lzma_easy_buffer_encode: one Block over the whole input ----
    def stream_buffer_encode(self, data, preset=6, check=LZMA_CHECK_CRC64, opts=None, n=None):
        o = opts if opts is not None else lzma_lzma_preset(preset)
        n = len(data) if n is None else n
        cap = lib().xzb_stream_buffer_bound(n)
        out = (C.c_uint8 * cap)()
        sp, _k1 = _ptr(data)
        sz = C.c_uint64()
        r = lib().xzb_stream_buffer_encode(self._h, sp, n, C.byref(o), check, out, cap, C.byref(sz))
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return bytes(out[: sz.value])

    # ---- one Block piece by piece in bounded memory (xzb_block_decoder_*) ----
    def block_decoder(self, header, check, flags=0):
        """A resumable decoder of one LZMA2 Block whose whole Block Header is `header` in a Stream with Check ID `check`;
        see BlockDecoder."""
        return BlockDecoder(self, header, check, flags)

    # ---- lzma_stream_buffer_decode (one Stream): returns (ret, bytes, input bytes used) ----
    def stream_buffer_decode(self, data, cap, flags=0):
        out = (C.c_uint8 * max(cap, 1))()
        sp, _k1 = _ptr(data)
        sz = C.c_uint64(); used = C.c_uint64()
        r = lib().xzb_stream_buffer_decode(self._h, sp, len(data), out, cap, C.byref(sz), C.byref(used), flags)
        return r, bytes(out[: sz.value]), used.value

    # ---- batches of independent whole Streams (xzb_stream_encode_batch[_device]) ----
    def stream_encode_batch(self, items, preset=6, block_size=0, check=LZMA_CHECK_CRC64, opts=None, caps=None):
        """One lzma_stream_encoder_mt Stream per item (what stream_encode gives it alone), all in one call:
        [(ret, Stream bytes)] in item order.  caps[i] (default xzb_stream_bound of the item's size at the effective
        Block size) is item i's output room."""
        o = opts if opts is not None else lzma_lzma_preset(preset)
        n = len(items)
        views = [bytes(x) for x in items]
        sizes = [len(v) for v in views]
        bs = block_size if block_size else max(3 * o.dict_size, 1 << 20)
        caps = [stream_bound(s, bs) for s in sizes] if caps is None else list(caps)
        src = bytearray(b"".join(views)) or bytearray(1)
        A = C.c_uint64 * max(n, 1)
        in_off, out_off = A(), A()
        for i in range(1, n):
            in_off[i] = in_off[i - 1] + sizes[i - 1]
            out_off[i] = out_off[i - 1] + caps[i - 1]
        out = (C.c_uint8 * max(sum(caps), 1))()
        size, rets = A(), (C.c_uint32 * max(n, 1))()
        sp, _k = _ptr(src)
        r = lib().xzb_stream_encode_batch(self._h, n, sp, in_off, A(*sizes), C.byref(o), check, block_size, out, out_off, A(*caps), size,
                                          rets)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        raw = memoryview(out).cast("B")   # batches of several GiB: no C.string_at (its size is an int)
        return [(rets[i], bytes(raw[out_off[i]: out_off[i] + size[i]])) for i in range(n)]

    def stream_encode_batch_device(self, d_in, in_off, in_size, opts, check, block_size, d_out, out_off, out_cap):
        """The whole-Stream batch on device memory: d_in / d_out are addresses (or CUDA tensors; synchronise their stream
        first), the offset and size lists stay on the host.  Returns [(ret, Stream size)]; the Streams are at
        d_out + out_off[i]."""
        n = len(in_off)
        A = C.c_uint64 * max(n, 1)
        size, rets = A(), (C.c_uint32 * max(n, 1))()
        ip, _k1 = _ptr(d_in)
        op, _k2 = _ptr(d_out)
        r = lib().xzb_stream_encode_batch_device(self._h, n, ip, A(*in_off), A(*in_size), C.byref(opts), check, block_size, op, A(*out_off),
                                                 A(*out_cap), size, rets)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return [(rets[i], size[i]) for i in range(n)]

    # ---- batches of independent one-shot Streams (xzb_stream_buffer_*_batch) ----
    def stream_buffer_encode_batch(self, items, preset=6, check=LZMA_CHECK_CRC64, opts=None, caps=None):
        """One lzma_stream_buffer_encode per item, all in one call: [(ret, Stream bytes)] in item order.
        caps[i] (default xzb_stream_buffer_bound of the item's size) is item i's output room."""
        o = opts if opts is not None else lzma_lzma_preset(preset)
        n = len(items)
        views = [bytes(x) for x in items]
        sizes = [len(v) for v in views]
        caps = [lib().xzb_stream_buffer_bound(s) for s in sizes] if caps is None else list(caps)
        src = bytearray(b"".join(views)) or bytearray(1)
        A = C.c_uint64 * max(n, 1)
        in_off, out_off = A(), A()
        for i in range(1, n):
            in_off[i] = in_off[i - 1] + sizes[i - 1]
            out_off[i] = out_off[i - 1] + caps[i - 1]
        out = (C.c_uint8 * max(sum(caps), 1))()
        size, rets = A(), (C.c_uint32 * max(n, 1))()
        sp, _k = _ptr(src)
        r = lib().xzb_stream_buffer_encode_batch(self._h, n, sp, in_off, A(*sizes), C.byref(o), check, out, out_off, A(*caps), size, rets)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        raw = memoryview(out).cast("B")   # batches of several GiB: no C.string_at (its size is an int)
        return [(rets[i], bytes(raw[out_off[i]: out_off[i] + size[i]])) for i in range(n)]

    def stream_buffer_encode_batch_device(self, d_in, in_off, in_size, opts, check, d_out, out_off, out_cap):
        """The batch on device memory: d_in / d_out are addresses (or CUDA tensors; synchronise their stream first),
        the offset and size lists stay on the host.  Returns [(ret, Stream size)]; the Streams are at d_out + out_off[i]."""
        n = len(in_off)
        A = C.c_uint64 * max(n, 1)
        size, rets = A(), (C.c_uint32 * max(n, 1))()
        ip, _k1 = _ptr(d_in)
        op, _k2 = _ptr(d_out)
        r = lib().xzb_stream_buffer_encode_batch_device(self._h, n, ip, A(*in_off), A(*in_size), C.byref(opts), check, op, A(*out_off),
                                                        A(*out_cap), size, rets)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return [(rets[i], size[i]) for i in range(n)]

    def stream_buffer_decode_batch(self, streams, caps, flags=0):
        """One lzma_stream_buffer_decode per Stream, all in one call: [(ret, bytes, input bytes used)] in Stream order."""
        n = len(streams)
        views = [bytes(x) for x in streams]
        src = bytearray(b"".join(views)) or bytearray(1)
        A = C.c_uint64 * max(n, 1)
        in_off, out_off = A(), A()
        for i in range(1, n):
            in_off[i] = in_off[i - 1] + len(views[i - 1])
            out_off[i] = out_off[i - 1] + caps[i - 1]
        out = (C.c_uint8 * max(sum(caps), 1))()
        size, used, rets = A(), A(), (C.c_uint32 * max(n, 1))()
        sp, _k = _ptr(src)
        r = lib().xzb_stream_buffer_decode_batch(self._h, n, sp, in_off, A(*[len(v) for v in views]), out, out_off, A(*caps), size, used,
                                                 rets, flags)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        raw = C.string_at(out, len(out))
        return [(rets[i], raw[out_off[i]: out_off[i] + size[i]], used[i]) for i in range(n)]

    def stream_buffer_decode_batch_device(self, d_in, in_off, in_size, d_out, out_off, out_cap, flags=0):
        """The decode batch on device memory: d_in / d_out are addresses (or CUDA tensors; synchronise their stream
        first), the offset and size lists stay on the host.  Returns [(ret, output size, input bytes used)]; item i's
        output is at d_out + out_off[i]."""
        n = len(in_off)
        A = C.c_uint64 * max(n, 1)
        size, used, rets = A(), A(), (C.c_uint32 * max(n, 1))()
        ip, _k1 = _ptr(d_in)
        op, _k2 = _ptr(d_out)
        r = lib().xzb_stream_buffer_decode_batch_device(self._h, n, ip, A(*in_off), A(*in_size), op, A(*out_off), A(*out_cap), size,
                                                        used, rets, flags)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return [(rets[i], size[i], used[i]) for i in range(n)]

    # ---- lzma_stream_decoder + lzma_code(FINISH) on host buffers ----
    def stream_decode_into(self, src, n, dst, cap):
        sp, _k1 = _ptr(src)
        dp, _k2 = _ptr(dst)
        sz = C.c_uint64()
        r = lib().xzb_stream_decode(self._h, sp, n, dp, cap, C.byref(sz))
        return r, sz.value

    def stream_decode(self, data, cap):
        out = (C.c_uint8 * max(cap, 1))()
        r, size = self.stream_decode_into(data, len(data), out, cap)
        return r, bytes(out[:size])

    # ---- device-resident block batches (the worker_encode / worker_decoder cut) ----
    def encode_blocks_device(self, d_in, n, opts, check, block_size, d_out, cap):
        nblocks = (n + block_size - 1) // block_size
        recs = (IndexRecord * max(nblocks, 1))()
        sz = C.c_uint64()
        r = lib().xzb_encode_blocks_device(self._h, d_in, n, C.byref(opts), check, block_size, d_out, cap, C.byref(sz), recs)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return sz.value, [(recs[i].unpadded_size, recs[i].uncompressed_size) for i in range(nblocks)]

    def encode_blocks_host(self, src, n, opts, check, block_size, dst, cap):
        """Host-buffer variant of encode_blocks_device (one rank's shard of Blocks)."""
        nblocks = (n + block_size - 1) // block_size
        recs = (IndexRecord * max(nblocks, 1))()
        sz = C.c_uint64()
        sp, _k1 = _ptr(src)
        dp, _k2 = _ptr(dst)
        r = lib().xzb_encode_blocks_host(self._h, sp, n, C.byref(opts), check, block_size, dp, cap, C.byref(sz), recs)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return sz.value, [(recs[i].unpadded_size, recs[i].uncompressed_size) for i in range(nblocks)]

    def decode_blocks_device(self, d_in, comp_off, comp_size, uncomp_size, out_off, dict_size, check, d_out):
        nb = len(comp_off)
        A64 = C.c_uint64 * nb
        rets = (C.c_uint32 * nb)()
        crcs = (C.c_uint64 * nb)()
        r = lib().xzb_decode_blocks_device(self._h, d_in, A64(*comp_off), A64(*comp_size), A64(*uncomp_size), A64(*out_off),
                                           (C.c_uint32 * nb)(*dict_size), nb, check, d_out, rets, crcs)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return list(rets), list(crcs)

    # ---- device memory helpers ----
    def device_alloc(self, size):
        p = C.c_void_p()
        r = lib().xzb_device_alloc(self._h, C.byref(p), size)
        if r != LZMA_OK:
            raise XzError(r, self._err())
        return p.value

    def device_free(self, p):
        lib().xzb_device_free(self._h, p)

    def h2d(self, d_dst, src, n):
        sp, _k = _ptr(src)
        r = lib().xzb_memcpy_h2d(self._h, d_dst, sp, n)
        if r != LZMA_OK:
            raise XzError(r, self._err())

    def d2h(self, dst, d_src, n):
        dp, _k = _ptr(dst)
        r = lib().xzb_memcpy_d2h(self._h, dp, d_src, n)
        if r != LZMA_OK:
            raise XzError(r, self._err())


class BlockDecoder:
    """xzb_block_decoder: .code(data, out_cap, finish) takes the whole LZMA2 chunks at the front of `data` (all of it
    when finish), then the Block Padding and Check field, and returns (ret, bytes, in_used): ret 0 = call again with
    the rest of the input (data[in_used:] first) or more room, 1 = the Block ended and every byte was handed out, else
    the lzma_ret of the error (the bytes decoded before it come first).  .record() is the Block's Index record
    (unpadded size, uncompressed size) after ret 1."""

    def __init__(self, ctx, header, check, flags=0):
        self._ctx = ctx
        self._h = C.c_void_p()
        hp, _k = _ptr(bytes(header))
        r = lib().xzb_block_decoder_create(ctx._h, hp, len(header), check, flags, C.byref(self._h))
        if r != LZMA_OK:
            raise XzError(r, ctx._err())

    def code(self, data, out_cap, finish=False):
        out = (C.c_uint8 * max(out_cap, 1))()
        dp, _k = _ptr(bytes(data) if data else b"\0")
        used, size = C.c_uint64(), C.c_uint64()
        r = lib().xzb_block_decoder_code(self._h, dp, len(data), C.byref(used), out, out_cap, C.byref(size), 1 if finish else 0)
        return r, bytes(out[: size.value]), used.value

    def code_into(self, src, n, dst, cap, finish=False):
        """The same on caller-owned buffers (addresses or objects _ptr takes): (ret, bytes written, in_used)."""
        sp, _k1 = _ptr(src)
        dp, _k2 = _ptr(dst)
        used, size = C.c_uint64(), C.c_uint64()
        r = lib().xzb_block_decoder_code(self._h, sp, n, C.byref(used), dp, cap, C.byref(size), 1 if finish else 0)
        return r, size.value, used.value

    def record(self):
        rec = IndexRecord()
        r = lib().xzb_block_decoder_record(self._h, C.byref(rec))
        if r != LZMA_OK:
            raise XzError(r, "the Block has not ended")
        return rec.unpadded_size, rec.uncompressed_size

    def stats(self):
        s = BlockDecoderStats()
        lib().xzb_block_decoder_stats(self._h, C.byref(s))
        return s

    def close(self):
        if self._h:
            lib().xzb_block_decoder_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def index_encode(records):
    """Index field for the given (unpadded, uncompressed) records (index_encoder.c:43-165)."""
    n = len(records)
    arr = (IndexRecord * max(n, 1))()
    for i, (u, v) in enumerate(records):
        arr[i].unpadded_size, arr[i].uncompressed_size = u, v
    size = lib().xzb_index_encode(arr, C.c_uint64(n), None)
    out = (C.c_uint8 * size)()
    lib().xzb_index_encode(arr, C.c_uint64(n), out)
    return bytes(out)


def stream_header(check):
    out = (C.c_uint8 * 12)()
    lib().xzb_stream_header_encode(out, C.c_uint32(check))
    return bytes(out)


def stream_footer(check, index_size):
    out = (C.c_uint8 * 12)()
    lib().xzb_stream_footer_encode(out, C.c_uint32(check), C.c_uint64(index_size))
    return bytes(out)
