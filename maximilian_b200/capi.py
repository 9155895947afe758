"""ctypes binding of libmaxib200.so (include/maxib200.h) -- the C ABI is the product boundary; this
module only marshals numpy / raw device pointers into it. There is no CPU implementation behind these
classes: a missing library or a missing CUDA device raises.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libmaxib200.so")

MEM_HOST, MEM_DEVICE, MEM_SPLIT, MEM_ASYNC = 0, 1, 2, 0x100
F64, F32 = 0, 1

OSC = dict(sinewave=0, coswave=1, phasor=2, saw=3, square=4, pulse=5, impulse=6, triangle=7, phasorbetween=8)
FILT = dict(none=0, lores=1, hires=2, svf=3, biquad=4)
BIQUAD = dict(lowpass=0, highpass=1, bandpass=2, notch=3, peak=4, lowshelf=5, highshelf=6)
P = dict(freq=0, phase=1, duty=2, cutoff=3, resonance=4, gain=5, env_attack=6, env_decay=7,
         env_sustain=8, env_release=9, env_holdtime=10, delay_size=11, delay_feedback=12, pan=13, delay_position=14,
         phasor_start=15, phasor_end=16, filt0=32, filt1=33, filt2=34, env_amplitude=35, env_output=36, env_holdcount=37,
         env_flags=38, delay_phase=39, osc_output=40)

EXPORTS = [
    "mxb_last_error", "mxb_version", "mxb_ctx_create", "mxb_ctx_destroy", "mxb_ctx_sample_rate",
    "mxb_ctx_synchronize", "mxb_host_alloc", "mxb_host_free",
    "mxb_bank_create", "mxb_bank_destroy", "mxb_bank_voices", "mxb_bank_set_param", "mxb_bank_set_param_async", "mxb_bank_get_state",
    "mxb_bank_get_ring", "mxb_bank_set_state", "mxb_bank_set_ring", "mxb_bank_clone", "mxb_bank_process", "mxb_bank_process_fm", "mxb_bank_process_mod", "mxb_play_block", "mxb_bank_launch_count", "mxb_env_coeffs",
    "mxb_exchange_create", "mxb_exchange_local_handle", "mxb_exchange_connect", "mxb_exchange_status", "mxb_exchange_destroy", "mxb_bank_set_exchange", "mxb_patch_set_exchange",
    "mxb_stft_create", "mxb_stft_destroy", "mxb_stft_process", "mxb_stft_process2", "mxb_stft_launch_count",
    "mxb_mfcc_create", "mxb_mfcc_destroy", "mxb_mfcc_process",
    "mxb_istft_create", "mxb_istft_destroy", "mxb_istft_process",
    "mxb_octave_create", "mxb_octave_destroy", "mxb_octave_n_averages", "mxb_octave_config", "mxb_stft_process3",
    "mxb_ctx_set_tables", "mxb_patch_create", "mxb_patch_destroy", "mxb_patch_set_param", "mxb_patch_set_state", "mxb_patch_get_state",
    "mxb_patch_get_ring", "mxb_patch_process", "mxb_patch_launch_count", "mxb_patch_set_mode", "mxb_patch_get_mode", "mxb_patch_codegen",
    "mxb_patch_create2", "mxb_patch_get_held", "mxb_patch_set_held",
    "mxb_octave_process", "mxb_bark_create", "mxb_bark_destroy", "mxb_bark_process",
    "mxb_stft_process_ragged", "mxb_stft_get_pos", "mxb_istft_process_ragged",
]


class MxbError(RuntimeError):
    pass


class BankDesc(C.Structure):
    _fields_ = [("voices", C.c_int32), ("osc_kind", C.c_int32), ("filt_kind", C.c_int32),
                ("biquad_type", C.c_int32), ("env_kind", C.c_int32), ("delay_taps", C.c_int32),
                ("max_frames", C.c_int32), ("delay_mode", C.c_int32), ("svf_mix", C.c_double * 4)]


class Modulation(C.Structure):
    _fields_ = [("freq_tv", C.c_void_p), ("cutoff_tv", C.c_void_p), ("delay_size_tv", C.c_void_p), ("trig_tv", C.c_void_p)]


class StftOutputs(C.Structure):
    _fields_ = [("mags", C.c_void_p), ("phases", C.c_void_p), ("re", C.c_void_p), ("im", C.c_void_p),
                ("mags_db", C.c_void_p), ("flatness", C.c_void_p), ("centroid", C.c_void_p), ("coeffs", C.c_void_p)]


ENV_KIND = {False: 0, None: 0, True: 1, "adsr": 1, "ar": 2}          # maxiEnv::adsr / maxiEnv::ar
DELAY_MODE = {False: 0, None: 0, True: 0, "dl": 0, "position": 1}    # maxiDelayline::dl / dlFromPosition


_lib = None


def lib():
    """Load libmaxib200.so; raises if it has not been built (python -m maximilian_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MxbError(f"{LIB_PATH} is missing: build it with `python -m maximilian_b200.build` "
                       "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    pp = C.POINTER(C.c_void_p)
    sig = {
        "mxb_last_error": (C.c_char_p, []),
        "mxb_version": (i32, []),
        "mxb_ctx_create": (i32, [i32, i32, pp]),
        "mxb_ctx_destroy": (i32, [vp]),
        "mxb_ctx_sample_rate": (i32, [vp]),
        "mxb_ctx_synchronize": (i32, [vp]),
        "mxb_host_alloc": (i32, [vp, C.c_uint64, pp]),
        "mxb_host_free": (i32, [vp, vp]),
        "mxb_bank_create": (i32, [vp, C.POINTER(BankDesc), pp]),
        "mxb_bank_destroy": (i32, [vp]),
        "mxb_bank_voices": (i32, [vp]),
        "mxb_bank_set_param": (i32, [vp, i32, vp, i32]),
        "mxb_bank_set_param_async": (i32, [vp, i32, vp, i32, vp]),
        "mxb_bank_get_state": (i32, [vp, i32, vp, i32]),
        "mxb_bank_get_ring": (i32, [vp, i32, vp, i32, i32]),
        "mxb_bank_set_state": (i32, [vp, i32, vp, i32]),
        "mxb_bank_set_ring": (i32, [vp, i32, vp, i32, i32]),
        "mxb_bank_clone": (i32, [vp, pp]),
        "mxb_bank_process": (i32, [vp, i32, vp, vp, vp, i32, vp, i32, vp]),
        "mxb_bank_process_fm": (i32, [vp, i32, vp, vp, vp, vp, i32, vp, i32, vp]),
        "mxb_bank_process_mod": (i32, [vp, i32, C.POINTER(Modulation), vp, vp, vp, i32, vp, i32, vp]),
        "mxb_play_block": (i32, [vp, vp, i32, i32]),
        "mxb_bank_launch_count": (i64, [vp]),
        "mxb_env_coeffs": (i32, [i32, vp, i64, i32, vp]),
        "mxb_exchange_create": (i32, [vp, i32, i32, i32, pp]),
        "mxb_exchange_local_handle": (i32, [vp, vp, i32]),
        "mxb_exchange_connect": (i32, [vp, vp]),
        "mxb_exchange_status": (i32, [vp, C.POINTER(i32)]),
        "mxb_exchange_destroy": (i32, [vp]),
        "mxb_bank_set_exchange": (i32, [vp, vp]),
        "mxb_patch_set_exchange": (i32, [vp, vp]),
        "mxb_stft_create": (i32, [vp, i32, i32, i32, pp]),
        "mxb_stft_destroy": (i32, [vp]),
        "mxb_stft_process": (i32, [vp, vp, i64, i64, i32, i32, vp, vp, vp, vp, vp, vp, C.POINTER(i32), i32, vp]),
        "mxb_stft_process2": (i32, [vp, vp, i64, i64, i32, i32, C.POINTER(StftOutputs), vp, C.POINTER(i32), i32, vp]),
        "mxb_stft_launch_count": (i64, [vp]),
        "mxb_mfcc_create": (i32, [vp, i32, i32, i32, dbl, dbl, pp]),
        "mxb_mfcc_destroy": (i32, [vp]),
        "mxb_mfcc_process": (i32, [vp, vp, i64, vp, vp, i32, vp]),
        "mxb_istft_create": (i32, [vp, i32, i32, i32, pp]),
        "mxb_istft_destroy": (i32, [vp]),
        "mxb_istft_process": (i32, [vp, vp, vp, i32, vp, i32, vp]),
        "mxb_octave_create": (i32, [vp, i32, C.c_float, i32, i32, pp]),
        "mxb_octave_destroy": (i32, [vp]),
        "mxb_octave_n_averages": (i32, [vp]),
        "mxb_octave_config": (i32, [vp, i32, C.c_float, C.c_float, C.c_float]),
        "mxb_stft_process3": (i32, [vp, vp, i64, i64, i32, i32, C.POINTER(StftOutputs), vp, vp, C.POINTER(i32), i32, vp]),
        "mxb_ctx_set_tables": (i32, [vp, vp, vp, dbl]),
        "mxb_patch_create": (i32, [vp, vp, pp]),
        "mxb_patch_destroy": (i32, [vp]),
        "mxb_patch_set_param": (i32, [vp, i32, vp, i32]),
        "mxb_patch_set_state": (i32, [vp, i32, i32, vp, i32]),
        "mxb_patch_get_state": (i32, [vp, i32, i32, vp, i32]),
        "mxb_patch_get_ring": (i32, [vp, i32, i32, vp, i32, i32]),
        "mxb_patch_process": (i32, [vp, i32, vp, vp, vp, i32, vp]),
        "mxb_patch_launch_count": (i64, [vp]),
        "mxb_patch_set_mode": (i32, [vp, i32]),
        "mxb_patch_get_mode": (i32, [vp]),
        "mxb_patch_codegen": (i32, [vp, vp, i64, vp, i32]),
        "mxb_patch_create2": (i32, [vp, vp, i32, vp, pp]),
        "mxb_patch_get_held": (i32, [vp, i32, vp, i32]),
        "mxb_patch_set_held": (i32, [vp, i32, vp, i32]),
        "mxb_octave_process": (i32, [vp, vp, i32, i32, vp, vp, i32, vp]),
        "mxb_bark_create": (i32, [vp, i32, i32, pp]),
        "mxb_bark_destroy": (i32, [vp]),
        "mxb_bark_process": (i32, [vp, vp, i64, vp, vp, vp, i32, vp]),
        "mxb_stft_process_ragged": (i32, [vp, vp, i64, i64, vp, i32, C.POINTER(StftOutputs), vp, vp, vp, i32, vp]),
        "mxb_stft_get_pos": (i32, [vp, vp]),
        "mxb_istft_process_ragged": (i32, [vp, vp, vp, vp, i32, vp, i32, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(L, name)          # AttributeError here = the library does not export a declared symbol
        fn.restype, fn.argtypes = res, args
    _lib = L
    return L


def check(rc, what=""):
    if rc != 0:
        raise MxbError(f"{what} -> {rc}: {lib().mxb_last_error().decode(errors='replace')}")


def _np_ptr(a):
    return C.c_void_p(a.ctypes.data) if a is not None else None


def _ptr(x):
    """numpy array -> host pointer; int -> raw (device) pointer; None -> NULL."""
    if x is None:
        return None
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    return C.c_void_p(int(x))


class Context:
    """mxb_ctx: one CUDA device + the sample rate (the reference's maxiSettings::setup)."""

    def __init__(self, device=0, sample_rate=48000):
        self.h = C.c_void_p()
        check(lib().mxb_ctx_create(device, sample_rate, C.byref(self.h)), "mxb_ctx_create")
        self.device, self.sample_rate = device, sample_rate

    def synchronize(self):
        check(lib().mxb_ctx_synchronize(self.h), "mxb_ctx_synchronize")

    def close(self):
        if self.h:
            lib().mxb_ctx_destroy(self.h)
            self.h = None


_default_ctx = {}


def default_context(device=0, sample_rate=48000):
    key = (device, sample_rate)
    if key not in _default_ctx:
        _default_ctx[key] = Context(device, sample_rate)
    return _default_ctx[key]


class Bank:
    """V voices of  osc -> [adsr] -> [filter] -> [delay] -> out / stereo mix  on the GPU (mxb_bank)."""

    def __init__(self, voices, osc="saw", filt="none", env=False, delay=False, sample_rate=48000,
                 biquad_type="lowpass", svf_mix=(1.0, 0.0, 0.0, 0.0), delay_capacity=4096, max_frames=1024,
                 ctx=None, device=0):
        self.ctx = ctx or default_context(device, sample_rate)
        if self.ctx.sample_rate != sample_rate:
            raise MxbError("context sample rate differs from the requested one")
        self.V = int(voices)
        self.max_frames = int(max_frames)
        d = BankDesc(self.V, OSC[osc], FILT[filt], BIQUAD[biquad_type], ENV_KIND[env],
                     int(delay_capacity) if delay else 0, self.max_frames, DELAY_MODE[delay], (C.c_double * 4)(*svf_mix))
        self.h = C.c_void_p()
        check(lib().mxb_bank_create(self.ctx.h, C.byref(d), C.byref(self.h)), "mxb_bank_create")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_bank_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- parameters / state ------------------------------------------------------------------
    def set(self, name, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        check(lib().mxb_bank_set_param(self.h, P[name], _np_ptr(a), MEM_HOST), f"mxb_bank_set_param({name})")

    def set_device(self, name, dev_ptr):
        check(lib().mxb_bank_set_param(self.h, P[name], C.c_void_p(int(dev_ptr)), MEM_DEVICE), f"mxb_bank_set_param({name})")

    def get(self, name):
        a = np.empty(self.V, dtype=np.float64)
        check(lib().mxb_bank_get_state(self.h, P[name], _np_ptr(a), MEM_HOST), f"mxb_bank_get_state({name})")
        return a

    def ring(self, v, n):
        a = np.empty(n, dtype=np.float64)
        check(lib().mxb_bank_get_ring(self.h, v, _np_ptr(a), n, MEM_HOST), "mxb_bank_get_ring")
        return a

    def set_state(self, name, values):
        """mxb_bank_set_state: one MXB_S_* array (filt0.., env_*, delay_phase, osc_output)."""
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        check(lib().mxb_bank_set_state(self.h, P[name], _np_ptr(a), MEM_HOST), f"mxb_bank_set_state({name})")

    def set_ring(self, v, values):
        a = np.ascontiguousarray(values, dtype=np.float64)
        check(lib().mxb_bank_set_ring(self.h, v, _np_ptr(a), a.size, MEM_HOST), "mxb_bank_set_ring")

    def clone(self):
        """mxb_bank_clone: a deep copy (parameters, coefficients, state, rings) on the same context."""
        other = object.__new__(Bank)
        other.ctx, other.V, other.max_frames = self.ctx, self.V, self.max_frames
        other.h = C.c_void_p()
        check(lib().mxb_bank_clone(self.h, C.byref(other.h)), "mxb_bank_clone")
        return other

    @property
    def launches(self):
        return int(lib().mxb_bank_launch_count(self.h))

    # -- one block ---------------------------------------------------------------------------
    def process(self, nframes, trig_on=None, trig_off=None, want_out=True, want_mix=False, out_dtype=np.float64,
                out=None, mix=None, freq_tv=None, cutoff_tv=None, delay_size_tv=None, trig_tv=None):
        """Host buffers in, host buffers out (MXB_MEM_HOST). Returns (out[nframes][V] | None, mix[nframes][2] | None).
        freq_tv / cutoff_tv / delay_size_tv: optional per-sample oscillator frequency / filter cutoff / delay size [nframes][V]
        (mxb_bank_process_mod)."""
        if freq_tv is not None or cutoff_tv is not None or delay_size_tv is not None or trig_tv is not None:
            tv = np.ascontiguousarray(trig_tv, dtype=np.uint8) if trig_tv is not None else None
            assert tv is None or tv.shape == (nframes, self.V)
            f = np.ascontiguousarray(freq_tv, dtype=np.float64) if freq_tv is not None else None
            cu = np.ascontiguousarray(cutoff_tv, dtype=np.float64) if cutoff_tv is not None else None
            assert f is None or f.shape == (nframes, self.V)
            assert cu is None or cu.shape == (nframes, self.V)
            ds = np.ascontiguousarray(delay_size_tv, dtype=np.float64) if delay_size_tv is not None else None
            assert ds is None or ds.shape == (nframes, self.V)
            mod = Modulation(_np_ptr(f), _np_ptr(cu), _np_ptr(ds), _np_ptr(tv))
            f32 = np.dtype(out_dtype) == np.float32
            if want_out and out is None:
                out = np.empty((nframes, self.V), dtype=np.float32 if f32 else np.float64)
            if want_mix and mix is None:
                mix = np.empty((nframes, 2), dtype=np.float64)
            ton = np.ascontiguousarray(trig_on, dtype=np.int32) if trig_on is not None else None
            toff = np.ascontiguousarray(trig_off, dtype=np.int32) if trig_off is not None else None
            check(lib().mxb_bank_process_mod(self.h, nframes, C.byref(mod), _np_ptr(ton), _np_ptr(toff),
                                             _np_ptr(out if want_out else None), F32 if f32 else F64,
                                             _np_ptr(mix if want_mix else None), MEM_HOST, None), "mxb_bank_process_mod")
            return (out if want_out else None), (mix if want_mix else None)
        f32 = np.dtype(out_dtype) == np.float32
        if want_out and out is None:
            out = np.empty((nframes, self.V), dtype=np.float32 if f32 else np.float64)
        if want_mix and mix is None:
            mix = np.empty((nframes, 2), dtype=np.float64)
        ton = np.ascontiguousarray(trig_on, dtype=np.int32) if trig_on is not None else None
        toff = np.ascontiguousarray(trig_off, dtype=np.int32) if trig_off is not None else None
        check(lib().mxb_bank_process(self.h, nframes, _np_ptr(ton), _np_ptr(toff), _np_ptr(out if want_out else None),
                                     F32 if f32 else F64, _np_ptr(mix if want_mix else None), MEM_HOST, None),
              "mxb_bank_process")
        return (out if want_out else None), (mix if want_mix else None)

    def play_block(self, nframes, channels=2):
        """mxb_play_block: the interleaved buffer an audio callback would hand to the driver."""
        buf = np.empty((nframes, channels), dtype=np.float64)
        check(lib().mxb_play_block(self.h, _np_ptr(buf), nframes, channels), "mxb_play_block")
        return buf

    def process_device(self, nframes, out_ptr=None, mix_ptr=None, trig_on_ptr=None, trig_off_ptr=None,
                       f32=False, stream=0):
        """Device pointers, asynchronous on `stream` (a raw cudaStream_t value)."""
        check(lib().mxb_bank_process(self.h, nframes, _ptr(trig_on_ptr), _ptr(trig_off_ptr), _ptr(out_ptr),
                                     F32 if f32 else F64, _ptr(mix_ptr), MEM_DEVICE, C.c_void_p(int(stream)) if stream else None),
              "mxb_bank_process")


    def process_mod_device(self, nframes, out_ptr=None, mix_ptr=None, freq_tv_ptr=None, cutoff_tv_ptr=None, delay_size_tv_ptr=None,
                           trig_tv_ptr=None, trig_on_ptr=None, trig_off_ptr=None, f32=False, stream=0):
        """mxb_bank_process_mod with device pointers throughout (per-sample arrays [nframes][V] resident on the device), asynchronous
        on `stream`."""
        mod = Modulation(_ptr(freq_tv_ptr), _ptr(cutoff_tv_ptr), _ptr(delay_size_tv_ptr), _ptr(trig_tv_ptr))
        check(lib().mxb_bank_process_mod(self.h, nframes, C.byref(mod), _ptr(trig_on_ptr), _ptr(trig_off_ptr), _ptr(out_ptr),
                                         F32 if f32 else F64, _ptr(mix_ptr), MEM_DEVICE, C.c_void_p(int(stream)) if stream else None),
              "mxb_bank_process_mod")

    def process_split(self, nframes, out_ptr, mix, trig_on=None, trig_off=None, f32=False, stream=0, wait=True):
        """MXB_MEM_SPLIT: gates / mix are host numpy arrays, `out_ptr` is a raw device pointer (or None).
        Returns when the mix is in host memory; with wait=False (MXB_MEM_ASYNC; page-locked host arrays) as soon as the
        block is enqueued -- the mix is valid after the stream / context has been synchronised."""
        check(lib().mxb_bank_process(self.h, nframes, _np_ptr(trig_on), _np_ptr(trig_off), _ptr(out_ptr),
                                     F32 if f32 else F64, _np_ptr(mix), MEM_SPLIT | (0 if wait else MEM_ASYNC),
                                     C.c_void_p(int(stream)) if stream else None),
              "mxb_bank_process")

    def set_host_array(self, name, a, stream=None):
        """set() without the broadcast/convert step: `a` must be a contiguous float64 array of V values.
        With `stream` (a raw cudaStream_t value; 0 = default stream) the copy is stream-ordered and asynchronous
        (mxb_bank_set_param_async; `a` should live in pinned memory)."""
        if stream is None:
            check(lib().mxb_bank_set_param(self.h, P[name], C.c_void_p(a.ctypes.data), MEM_HOST), f"mxb_bank_set_param({name})")
        else:
            check(lib().mxb_bank_set_param_async(self.h, P[name], C.c_void_p(a.ctypes.data), MEM_HOST,
                                                 C.c_void_p(int(stream)) if stream else None), f"mxb_bank_set_param_async({name})")


class Exchange:
    """mxb_exchange: peer-memory mix-bus exchange between the ranks of one box (one process per GPU)."""
    HANDLE_BYTES = 64

    def __init__(self, ctx, rank, world, max_doubles=2 * 1024):
        self.ctx, self.rank, self.world = ctx, rank, world
        self.h = C.c_void_p()
        check(lib().mxb_exchange_create(ctx.h, rank, world, max_doubles, C.byref(self.h)), "mxb_exchange_create")

    def local_handle(self):
        buf = C.create_string_buffer(self.HANDLE_BYTES)
        check(lib().mxb_exchange_local_handle(self.h, buf, self.HANDLE_BYTES), "mxb_exchange_local_handle")
        return bytes(buf.raw)

    def connect(self, handles):
        """handles: list of `world` byte strings (rank order), as returned by every rank's local_handle()."""
        assert len(handles) == self.world
        blob = b"".join(handles)
        check(lib().mxb_exchange_connect(self.h, C.c_char_p(blob)), "mxb_exchange_connect")

    def connect_with_torch_distributed(self):
        """Exchange the IPC handles over an initialised torch.distributed process group."""
        import torch.distributed as dist
        handles = [None] * self.world
        dist.all_gather_object(handles, self.local_handle())
        self.connect(handles)
        dist.barrier()

    def status(self):
        """Bit mask of ranks whose contribution was missing from some bus (0 = all exchanges completed)."""
        m = C.c_int32(0)
        check(lib().mxb_exchange_status(self.h, C.byref(m)), "mxb_exchange_status")
        return m.value

    def attach(self, bank):
        """bank: a Bank or a Patch (its mix bus then leaves every block as the sum over all ranks)."""
        if isinstance(bank, Patch):
            check(lib().mxb_patch_set_exchange(bank.h, self.h), "mxb_patch_set_exchange")
        else:
            check(lib().mxb_bank_set_exchange(bank.h, self.h), "mxb_bank_set_exchange")
        bank._exchange = self

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_exchange_destroy(self.h)
            self.h = None


def env_coeffs(kind, ms, sample_rate=48000):
    """maxiEnv setters, vectorised: kind 0 setAttack, 1 setAttackMS, 2 setDecay/setRelease."""
    ms = np.ascontiguousarray(ms, dtype=np.float64)
    out = np.empty_like(ms)
    check(lib().mxb_env_coeffs(kind, _np_ptr(ms), ms.size, sample_rate, _np_ptr(out)), "mxb_env_coeffs")
    return out


class Stft:
    """Streaming STFT over C channels (mxb_stft), optionally fused with an Mfcc."""

    def __init__(self, channels, fft_size=1024, hop=512, ctx=None, device=0, sample_rate=48000):
        self.ctx = ctx or default_context(device, sample_rate)
        self.C, self.n, self.hop, self.bins = int(channels), int(fft_size), int(hop), int(fft_size) // 2
        self.h = C.c_void_p()
        check(lib().mxb_stft_create(self.ctx.h, self.C, self.n, self.hop, C.byref(self.h)), "mxb_stft_create")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_stft_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def launches(self):
        return int(lib().mxb_stft_launch_count(self.h))

    def process(self, x, want=("mags", "phases", "re", "im"), mfcc=None):
        """x: float32 [C][n] planar host array. Returns dict of [C][frames][bins] (+ 'mfcc' [C][frames][coeffs])."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        assert x.shape[0] == self.C
        n = x.shape[1]
        maxf = max(1, n // self.hop + 2)
        bufs = {k: (np.zeros((self.C, maxf, self.bins), dtype=np.float32) if k in want else None)
                for k in ("mags", "phases", "re", "im")}
        co = np.zeros((self.C, maxf, mfcc.coeffs), dtype=np.float64) if mfcc is not None else None
        nf = C.c_int32(0)
        check(lib().mxb_stft_process(self.h, _np_ptr(x), n, 1, n, maxf, _np_ptr(bufs["mags"]), _np_ptr(bufs["phases"]),
                                     _np_ptr(bufs["re"]), _np_ptr(bufs["im"]), mfcc.h if mfcc is not None else None,
                                     _np_ptr(co), C.byref(nf), MEM_HOST, None), "mxb_stft_process")
        f = nf.value
        r = {k: np.ascontiguousarray(v[:, :f]) for k, v in bufs.items() if v is not None}
        if co is not None:
            r["mfcc"] = np.ascontiguousarray(co[:, :f])
        return r

    def process_features(self, x):
        """x: float32 [C][n] planar host array -> dict(mags, mags_db [C][frames][bins]; flatness, centroid [C][frames]):
        maxiFFT::getMagnitudesDB / spectralFlatness / spectralCentroid fused into the transform (mxb_stft_process2)."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        n = x.shape[1]
        maxf = max(1, n // self.hop + 2)
        mags = np.zeros((self.C, maxf, self.bins), dtype=np.float32); db = np.zeros_like(mags)
        fl = np.zeros((self.C, maxf), dtype=np.float32); ce = np.zeros_like(fl)
        o = StftOutputs(mags.ctypes.data, None, None, None, db.ctypes.data, fl.ctypes.data, ce.ctypes.data, None)
        nf = C.c_int32(0)
        check(lib().mxb_stft_process2(self.h, _np_ptr(x), n, 1, n, maxf, C.byref(o), None, C.byref(nf), MEM_HOST, None), "mxb_stft_process2")
        f = nf.value
        return dict(mags=mags[:, :f].copy(), mags_db=db[:, :f].copy(), flatness=fl[:, :f].copy(), centroid=ce[:, :f].copy())

    def process_device(self, in_ptr, stride_c, stride_t, n, max_frames, mags=None, phases=None, re=None, im=None,
                       mfcc=None, coeffs=None, stream=0):
        nf = C.c_int32(0)
        check(lib().mxb_stft_process(self.h, _ptr(in_ptr), stride_c, stride_t, n, max_frames, _ptr(mags), _ptr(phases),
                                     _ptr(re), _ptr(im), mfcc.h if mfcc is not None else None, _ptr(coeffs),
                                     C.byref(nf), MEM_DEVICE, C.c_void_p(int(stream)) if stream else None), "mxb_stft_process")
        return nf.value

    def positions(self):
        """Each channel's maxiFFT::pos (mxb_stft_get_pos): int32 [C]."""
        pos = np.zeros(self.C, dtype=np.int32)
        check(lib().mxb_stft_get_pos(self.h, _np_ptr(pos)), "mxb_stft_get_pos")
        return pos

    def process_ragged(self, x, counts, want=("mags", "phases", "re", "im"), mfcc=None, octave=None, bark=False, features=False, max_frames=None):
        """Channels that advance independently (mxb_stft_process_ragged): channel c takes counts[c] samples of x[c] (float32 [C][>= max
        count] planar host array). Returns (frames int32 [C], dict of [C][max_frames][...] rows, channel c's first frames[c] of them
        valid): 'mags' / 'phases' / 're' / 'im' ([bins]), 'mags_db' / 'flatness' / 'centroid' with features, 'mfcc' with an Mfcc,
        'averages' / 'peaks' with an Octave, 'bark_specific' / 'bark_relative' / 'bark_total' with bark."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        if x.ndim != 2 or x.shape[0] != self.C or cnt.shape != (self.C,):
            raise MxbError(f"Stft.process_ragged: samples of shape {x.shape} and counts of shape {cnt.shape} for {self.C} channels")
        maxf = int(max_frames) if max_frames is not None else max(1, (self.n + int(cnt.max(initial=0))) // self.hop + 1)
        bins, C_ = self.bins, self.C
        names = list(want) + (["mags_db", "flatness", "centroid"] if features else [])
        r = {k: np.zeros((C_, maxf, bins) if k in ("mags", "phases", "re", "im", "mags_db") else (C_, maxf), dtype=np.float32) for k in names}
        if mfcc is not None:
            r["mfcc"] = np.zeros((C_, maxf, mfcc.coeffs))
        o = StftOutputs(*[r[k].ctypes.data if k in r else None for k in ("mags", "phases", "re", "im", "mags_db", "flatness", "centroid", "mfcc")])
        post = None
        if octave is not None or bark:
            if octave is not None:
                r["averages"] = np.zeros((C_, maxf, octave.n_averages), dtype=np.float32); r["peaks"] = np.zeros_like(r["averages"])
            if bark:
                r["bark_specific"] = np.zeros((C_, maxf, 24)); r["bark_relative"] = np.zeros_like(r["bark_specific"]); r["bark_total"] = np.zeros((C_, maxf))
            g = lambda k: r[k].ctypes.data if k in r else None
            post = StftPost(octave.h if octave is not None else None, g("averages"), g("peaks"), 1 if bark else 0,
                            g("bark_specific"), g("bark_relative"), g("bark_total"))
        nf = np.zeros(C_, dtype=np.int32)
        check(lib().mxb_stft_process_ragged(self.h, _np_ptr(x), x.shape[1], 1, _np_ptr(cnt), maxf, C.byref(o),
                                            C.byref(post) if post is not None else None, mfcc.h if mfcc is not None else None,
                                            _np_ptr(nf), MEM_HOST, None), "mxb_stft_process_ragged")
        return nf, r

    def process_ragged_device(self, in_ptr, stride_c, stride_t, counts, max_frames, mags=None, phases=None, re=None, im=None,
                              mfcc=None, coeffs=None, stream=0):
        """Device pointers (layouts of mxb_stft_process_ragged), asynchronous on `stream`; counts: host int array [C]. Returns frames [C]."""
        cnt = np.ascontiguousarray(counts, dtype=np.int32)
        o = StftOutputs(*[int(v) if v else None for v in (mags, phases, re, im, None, None, None, coeffs)])
        nf = np.zeros(self.C, dtype=np.int32)
        check(lib().mxb_stft_process_ragged(self.h, _ptr(in_ptr), stride_c, stride_t, _np_ptr(cnt), int(max_frames), C.byref(o), None,
                                            mfcc.h if mfcc is not None else None, _np_ptr(nf), MEM_DEVICE,
                                            C.c_void_p(int(stream)) if stream else None), "mxb_stft_process_ragged")
        return nf


class StftPost(C.Structure):
    _fields_ = [("octave", C.c_void_p), ("octave_averages", C.c_void_p), ("octave_peaks", C.c_void_p),
                ("bark", C.c_int32), ("bark_specific", C.c_void_p), ("bark_relative", C.c_void_p), ("bark_total", C.c_void_p)]


class Octave:
    """mxb_octave: maxiFFTOctaveAnalyzer::setup for every channel of one Stft (state: averages, peaks, hold times on the device). The
    state is shared by the transform's fused epilogue (stft_process_post) and process() on spectra in memory."""

    def __init__(self, channels, sampling_rate, n_bands, n_per_octave, ctx=None, device=0, sample_rate=48000):
        self.ctx = ctx or default_context(device, sample_rate)
        self.h = C.c_void_p()
        check(lib().mxb_octave_create(self.ctx.h, int(channels), float(sampling_rate), int(n_bands), int(n_per_octave), C.byref(self.h)), "mxb_octave_create")
        self.C, self.bands, self.n_averages = int(channels), int(n_bands), int(lib().mxb_octave_n_averages(self.h))

    def config(self, peak_hold_time=0, peak_decay_rate=0.9, eq_intercept=1.0, eq_slope=0.0):
        check(lib().mxb_octave_config(self.h, int(peak_hold_time), float(peak_decay_rate), float(eq_intercept), float(eq_slope)), "mxb_octave_config")

    def process(self, mags):
        """maxiFFTOctaveAnalyzer::calculate on every frame of float32 [C][frames][n_bands] host magnitudes, frames in order ->
        (averages, peaks) float32 [C][frames][nAverages] (mxb_octave_process)."""
        m = np.ascontiguousarray(mags, dtype=np.float32)
        if m.ndim != 3 or m.shape[0] != self.C or m.shape[2] != self.bands:
            raise MxbError(f"Octave.process: magnitudes of shape {m.shape}, expected ({self.C}, frames, {self.bands})")
        f = m.shape[1]
        av = np.zeros((self.C, f, self.n_averages), dtype=np.float32); pk = np.zeros_like(av)
        check(lib().mxb_octave_process(self.h, _np_ptr(m), f, f, _np_ptr(av), _np_ptr(pk), MEM_HOST, None), "mxb_octave_process")
        return av, pk

    def process_device(self, mags_ptr, frames, max_frames, averages_ptr=None, peaks_ptr=None, stream=0):
        """Device pointers (layout of mxb_octave_process), asynchronous on `stream` (a raw cudaStream_t value)."""
        check(lib().mxb_octave_process(self.h, _ptr(mags_ptr), int(frames), int(max_frames), _ptr(averages_ptr), _ptr(peaks_ptr), MEM_DEVICE,
                                       C.c_void_p(int(stream)) if stream else None), "mxb_octave_process")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_octave_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def stft_process_post(st, x, octave=None, bark=False):
    """Stft.process with the octave-analyser / Bark epilogues (mxb_stft_process3): x float32 [C][n] planar host array ->
    dict(mags [C][F][bins], averages / peaks [C][F][nAverages], bark_specific / bark_relative [C][F][24], bark_total [C][F])."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    n = x.shape[1]
    maxf = max(1, n // st.hop + 2)
    mags = np.zeros((st.C, maxf, st.bins), dtype=np.float32)
    o = StftOutputs(mags.ctypes.data, None, None, None, None, None, None, None)
    nA = octave.n_averages if octave is not None else 1
    av = np.zeros((st.C, maxf, nA), dtype=np.float32); pk = np.zeros_like(av)
    bs = np.zeros((st.C, maxf, 24)); br = np.zeros_like(bs); bt = np.zeros((st.C, maxf))
    post = StftPost(octave.h if octave is not None else None, av.ctypes.data if octave is not None else None, pk.ctypes.data if octave is not None else None,
                    1 if bark else 0, bs.ctypes.data if bark else None, br.ctypes.data if bark else None, bt.ctypes.data if bark else None)
    nf = C.c_int32(0)
    check(lib().mxb_stft_process3(st.h, _np_ptr(x), n, 1, n, maxf, C.byref(o), C.byref(post), None, C.byref(nf), MEM_HOST, None), "mxb_stft_process3")
    f = nf.value
    r = dict(mags=mags[:, :f].copy())
    if octave is not None:
        r.update(averages=av[:, :f].copy(), peaks=pk[:, :f].copy())
    if bark:
        r.update(bark_specific=bs[:, :f].copy(), bark_relative=br[:, :f].copy(), bark_total=bt[:, :f].copy())
    return r


class Bark:
    """mxb_bark: maxiBarkScaleAnalyser::setup(sample_rate, buffer_size) + specificLoudness / relativeLoudness / totalLoudness on any
    spectrum of buffer_size / 2 bins."""

    def __init__(self, sample_rate, buffer_size, ctx=None, device=0):
        self.ctx = ctx or default_context(device)           # the band limits come from sample_rate, not from the context's rate
        self.sample_rate, self.buffer_size, self.bins = int(sample_rate), int(buffer_size), int(buffer_size) // 2
        self.h = C.c_void_p()
        check(lib().mxb_bark_create(self.ctx.h, self.sample_rate, self.buffer_size, C.byref(self.h)), "mxb_bark_create")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_bark_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process(self, spectrum):
        """float32 [..., buffer_size / 2] host array -> (specific [..., 24], relative [..., 24], total [...]) float64."""
        m = np.ascontiguousarray(spectrum, dtype=np.float32)
        if m.ndim < 1 or m.shape[-1] != self.bins:
            raise MxbError(f"Bark.process: spectra of shape {m.shape}, expected (..., {self.bins})")
        lead = m.shape[:-1]
        n = int(np.prod(lead)) if lead else 1
        sp = np.empty((n, 24)); rl = np.empty((n, 24)); tt = np.empty(n)
        check(lib().mxb_bark_process(self.h, _np_ptr(m), n, _np_ptr(sp), _np_ptr(rl), _np_ptr(tt), MEM_HOST, None), "mxb_bark_process")
        return sp.reshape(lead + (24,)), rl.reshape(lead + (24,)), tt.reshape(lead)

    def process_device(self, spectrum_ptr, n, specific_ptr=None, relative_ptr=None, total_ptr=None, stream=0):
        """Device pointers (layout of mxb_bark_process), asynchronous on `stream` (a raw cudaStream_t value)."""
        check(lib().mxb_bark_process(self.h, _ptr(spectrum_ptr), int(n), _ptr(specific_ptr), _ptr(relative_ptr), _ptr(total_ptr), MEM_DEVICE,
                                     C.c_void_p(int(stream)) if stream else None), "mxb_bark_process")


class Mfcc:
    def __init__(self, num_bins=512, num_filters=42, num_coeffs=40, min_freq=20.0, max_freq=20000.0,
                 ctx=None, device=0, sample_rate=48000):
        self.ctx = ctx or default_context(device, sample_rate)
        self.bins, self.filters, self.coeffs = int(num_bins), int(num_filters), int(num_coeffs)
        self.h = C.c_void_p()
        check(lib().mxb_mfcc_create(self.ctx.h, self.bins, self.filters, self.coeffs, float(min_freq), float(max_freq),
                                    C.byref(self.h)), "mxb_mfcc_create")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_mfcc_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process(self, mags):
        m = np.ascontiguousarray(mags, dtype=np.float32)
        lead = m.shape[:-1]
        n = int(np.prod(lead)) if lead else 1
        co = np.empty((n, self.coeffs), dtype=np.float64)
        mb = np.empty((n, self.filters), dtype=np.float64)
        check(lib().mxb_mfcc_process(self.h, _np_ptr(m), n, _np_ptr(co), _np_ptr(mb), MEM_HOST, None), "mxb_mfcc_process")
        return co.reshape(lead + (self.coeffs,)), mb.reshape(lead + (self.filters,))


class Istft:
    def __init__(self, channels, fft_size=1024, hop=512, ctx=None, device=0, sample_rate=48000):
        self.ctx = ctx or default_context(device, sample_rate)
        self.C, self.n, self.hop, self.bins = int(channels), int(fft_size), int(hop), int(fft_size) // 2
        self.h = C.c_void_p()
        check(lib().mxb_istft_create(self.ctx.h, self.C, self.n, self.hop, C.byref(self.h)), "mxb_istft_create")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_istft_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def process(self, mags, phases):
        m = np.ascontiguousarray(mags, dtype=np.float32)
        p = np.ascontiguousarray(phases, dtype=np.float32)
        frames = m.shape[1]
        out = np.empty((self.C, frames * self.hop), dtype=np.float32)
        check(lib().mxb_istft_process(self.h, _np_ptr(m), _np_ptr(p), frames, _np_ptr(out), MEM_HOST, None), "mxb_istft_process")
        return out

    def process_ragged(self, mags, phases, frames):
        """Channels that advance independently (mxb_istft_process_ragged): channel c resynthesises the first frames[c] of its rows of
        float32 [C][max_frames][bins] mags / phases -> float32 [C][max_frames*hop], channel c's first frames[c]*hop samples valid."""
        m = np.ascontiguousarray(mags, dtype=np.float32)
        p = np.ascontiguousarray(phases, dtype=np.float32)
        fr = np.ascontiguousarray(frames, dtype=np.int32)
        if m.ndim != 3 or m.shape[0] != self.C or m.shape[2] != self.bins or p.shape != m.shape or fr.shape != (self.C,):
            raise MxbError(f"Istft.process_ragged: spectra of shape {m.shape} / {p.shape}, frames {fr.shape}")
        maxf = m.shape[1]
        out = np.zeros((self.C, maxf * self.hop), dtype=np.float32)
        check(lib().mxb_istft_process_ragged(self.h, _np_ptr(m), _np_ptr(p), _np_ptr(fr), maxf, _np_ptr(out), MEM_HOST, None),
              "mxb_istft_process_ragged")
        return out

    def process_ragged_device(self, mags_ptr, phases_ptr, frames, max_frames, out_ptr, stream=0):
        """Device pointers (layouts of mxb_istft_process_ragged), asynchronous on `stream`; frames: host int array [C]."""
        fr = np.ascontiguousarray(frames, dtype=np.int32)
        check(lib().mxb_istft_process_ragged(self.h, _ptr(mags_ptr), _ptr(phases_ptr), _np_ptr(fr), int(max_frames), _ptr(out_ptr), MEM_DEVICE,
                                             C.c_void_p(int(stream)) if stream else None), "mxb_istft_process_ragged")


# ------------------------------------------------------------------------------------------------ voice patches

class Stage(C.Structure):
    _fields_ = [("op", C.c_int32), ("kind", C.c_int32), ("dst", C.c_int32), ("reserved", C.c_int32), ("src", C.c_int32 * 8)]


class PatchDesc(C.Structure):
    _fields_ = [("voices", C.c_int32), ("n_stages", C.c_int32), ("n_params", C.c_int32), ("n_consts", C.c_int32), ("n_inputs", C.c_int32),
                ("max_frames", C.c_int32), ("delay_taps", C.c_int32), ("eg_stages", C.c_int32), ("eg_loop", C.c_int32), ("eg_retrigger", C.c_int32),
                ("stages", C.POINTER(Stage)), ("consts", C.POINTER(C.c_double)),
                ("eg_levels", C.POINTER(C.c_double)), ("eg_times", C.POINTER(C.c_double)), ("eg_curves", C.POINTER(C.c_double)),
                ("input_types", C.POINTER(C.c_int32))]


class Events(C.Structure):
    """mxb_events: one call's events of an MXB_IN_EVENTS stream (CSR by voice)"""
    _fields_ = [("first", C.c_void_p), ("frame", C.c_void_p), ("value", C.c_void_p)]


class EnvgenShape(C.Structure):
    _fields_ = [("stages", C.c_int32), ("loop", C.c_int32), ("retrigger", C.c_int32),
                ("levels", C.POINTER(C.c_double)), ("times", C.POINTER(C.c_double)), ("curves", C.POINTER(C.c_double))]


def _doubles(x):
    return (C.c_double * max(1, len(x)))(*x)


def envgen_shapes(shapes):
    """mxb_envgen_shape[] of (levels, times, curves, loop, retrigger) tuples; the second value keeps the arrays alive."""
    arr = (EnvgenShape * max(1, len(shapes)))()
    keep = [arr]
    for i, (lv, tm, cv, loop, retrig) in enumerate(shapes):
        a, b, c = _doubles(lv), _doubles(tm), _doubles(cv)
        arr[i] = EnvgenShape(len(tm), int(loop), int(retrig), a, b, c)
        keep += [a, b, c]
    return arr, keep


def set_tables(sine514, transition1001, sine_before, ctx=None, device=0, sample_rate=48000):
    """mxb_ctx_set_tables: the reference's sineBuffer / transition arrays (data of the reference, handed in by the caller)."""
    ctx = ctx or default_context(device, sample_rate)
    s = np.ascontiguousarray(sine514, dtype=np.float64); t = np.ascontiguousarray(transition1001, dtype=np.float64)
    assert s.size == 514 and t.size == 1001
    check(lib().mxb_ctx_set_tables(ctx.h, _np_ptr(s), _np_ptr(t), float(sine_before)), "mxb_ctx_set_tables")


PATCH_INTERPRET, PATCH_FUSED = 0, 1


def pack_bits(x):
    """[n][V] of 0 / 1 -> uint32 [n][(V + 31) / 32] (MXB_IN_BITS: voice v = bit v % 32 of word v / 32)"""
    x = np.asarray(x) != 0
    n, V = x.shape
    W = (V + 31) // 32
    pad = np.zeros((n, W * 32), dtype=np.uint8)
    pad[:, :V] = x
    return np.ascontiguousarray(np.packbits(pad, axis=1, bitorder="little")).view(np.uint32).reshape(n, W)


def pack_events(lists):
    """Per-voice lists of (frame, value) pairs -> the CSR triple of an events stream: first int32 [V + 1], frame int32 [n], value
    float64 [n]. Each voice's events keep their list order (the order in which they apply)."""
    first = np.zeros(len(lists) + 1, dtype=np.int32)
    first[1:] = np.cumsum([len(x) for x in lists])
    frame = np.array([f for x in lists for f, _ in x], dtype=np.int32)
    value = np.array([v for x in lists for _, v in x], dtype=np.float64)
    return first, frame, value


IN_TYPE = {"u8": 1, "bits": 2, "events": 3}      # MXB_IN_*; doubles (MXB_IN_F64 = 0) otherwise


def _patch_desc(defn, voices, max_frames, delay_taps):
    """mxb_patch_desc of a PatchDef; the second value keeps the ctypes arrays it points into alive."""
    st = (Stage * len(defn.stages))()
    for i, (op, kind, dst, src) in enumerate(defn.stages):
        st[i].op, st[i].kind, st[i].dst, st[i].reserved = op, kind, dst, 0
        for k in range(8):
            st[i].src[k] = src[k]
    consts = (C.c_double * max(1, len(defn.consts)))(*defn.consts)
    # one shape travels in the descriptor (mxb_patch_create); several go to mxb_patch_create2 (Patch) and the descriptor's eg_* stay empty
    eg = defn.eg if defn.eg is not None and len(defn.shapes) == 1 else ([0.0], [], [], False, False)
    lv = (C.c_double * max(1, len(eg[0])))(*eg[0]); tm = (C.c_double * max(1, len(eg[1])))(*eg[1]); cv = (C.c_double * max(1, len(eg[2])))(*eg[2])
    ty = (C.c_int32 * max(1, len(defn.inputs)))(*[IN_TYPE.get(defn.input_types.get(n), 0) for n in defn.inputs])
    d = PatchDesc(int(voices), len(defn.stages), len(defn.params), len(defn.consts), len(defn.inputs), int(max_frames), int(delay_taps),
                  len(eg[1]), int(eg[3]), int(eg[4]), st, consts, lv, tm, cv, ty)
    return d, (st, consts, lv, tm, cv, ty)


def patch_codegen(defn, compile=False):
    """mxb_patch_codegen: the CUDA source the library generates for this stage list (compile=True: also through NVRTC for
    sm_90a). Needs no device."""
    d, keep = _patch_desc(defn, 1, 1, 1)
    need = C.c_int64(0)
    check(lib().mxb_patch_codegen(C.byref(d), None, 0, C.byref(need), 0), "mxb_patch_codegen")
    buf = C.create_string_buffer(need.value)
    check(lib().mxb_patch_codegen(C.byref(d), buf, need.value, C.byref(need), 1 if compile else 0), "mxb_patch_codegen")
    return buf.value.decode()


class Patch:
    """mxb_patch: a per-voice signal graph (maximilian_b200.patchdef.PatchDef), run by the kernel the library generates and
    compiles for it (mode "fused", the default) or by the interpreting kernel (mode "interpret")."""

    def __init__(self, defn, voices, max_frames=1024, delay_taps=0, ctx=None, device=0, sample_rate=48000, mode=None):
        self.ctx = ctx or default_context(device, sample_rate)
        self.defn, self.V, self.max_frames = defn, int(voices), int(max_frames)
        d, keep = _patch_desc(defn, self.V, self.max_frames, delay_taps)
        self.h = C.c_void_p()
        if len(defn.shapes) <= 1:
            check(lib().mxb_patch_create(self.ctx.h, C.byref(d), C.byref(self.h)), "mxb_patch_create")
        else:
            shapes, keep_shapes = envgen_shapes(defn.shapes)
            check(lib().mxb_patch_create2(self.ctx.h, C.byref(d), len(defn.shapes), shapes, C.byref(self.h)), "mxb_patch_create2")
        if mode is not None:
            self.set_mode(mode)

    def set_mode(self, mode):
        m = {"interpret": PATCH_INTERPRET, "fused": PATCH_FUSED}.get(mode, mode)
        check(lib().mxb_patch_set_mode(self.h, int(m)), "mxb_patch_set_mode")

    @property
    def mode(self):
        return {PATCH_INTERPRET: "interpret", PATCH_FUSED: "fused"}[int(lib().mxb_patch_get_mode(self.h))]

    def process_device(self, nframes, input_ptrs, out_ptr, mix_ptr, stream=None):
        """device pointers in and out, asynchronous on `stream` (bench.py)"""
        ptrs = (C.c_void_p * max(1, len(input_ptrs)))(*input_ptrs)
        check(lib().mxb_patch_process(self.h, nframes, ptrs, C.c_void_p(out_ptr) if out_ptr else None, C.c_void_p(mix_ptr) if mix_ptr else None, MEM_DEVICE,
                                      C.c_void_p(stream) if stream else None), "mxb_patch_process")

    def close(self):
        if getattr(self, "h", None):
            lib().mxb_patch_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set(self, name, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        check(lib().mxb_patch_set_param(self.h, self.defn.params.index(name), _np_ptr(a), MEM_HOST), f"mxb_patch_set_param({name})")

    def get_state(self, stage, slot):
        a = np.empty(self.V, dtype=np.float64)
        check(lib().mxb_patch_get_state(self.h, stage, slot, _np_ptr(a), MEM_HOST), "mxb_patch_get_state")
        return a

    def set_state(self, stage, slot, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        check(lib().mxb_patch_set_state(self.h, stage, slot, _np_ptr(a), MEM_HOST), "mxb_patch_set_state")

    def ring(self, stage, v, n):
        a = np.empty(n, dtype=np.float64)
        check(lib().mxb_patch_get_ring(self.h, stage, v, _np_ptr(a), n, MEM_HOST), "mxb_patch_get_ring")
        return a

    def get_held(self, name):
        """the held values [V] of events stream `name`"""
        a = np.empty(self.V, dtype=np.float64)
        check(lib().mxb_patch_get_held(self.h, self.defn.inputs.index(name), _np_ptr(a), MEM_HOST), "mxb_patch_get_held")
        return a

    def set_held(self, name, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        check(lib().mxb_patch_set_held(self.h, self.defn.inputs.index(name), _np_ptr(a), MEM_HOST), "mxb_patch_set_held")

    @property
    def launches(self):
        return int(lib().mxb_patch_launch_count(self.h))

    def process(self, nframes, inputs=None, want_out=True, want_mix=False):
        """inputs: dict name -> float64 [nframes][V]; an events stream takes a CSR triple (first, frame, value) or per-voice lists of
        (frame, value) pairs (pack_events). Returns (out[nframes][V] | None, mix[nframes][2] | None)."""
        inputs = inputs or {}
        arrs, keep = [], []
        for n in self.defn.inputs:
            ty = self.defn.input_types.get(n)
            if ty == "events":
                x = inputs[n]
                first, frame, value = x if isinstance(x, tuple) and len(x) == 3 and isinstance(x[0], np.ndarray) else pack_events(x)
                first, frame = np.ascontiguousarray(first, dtype=np.int32), np.ascontiguousarray(frame, dtype=np.int32)
                value = np.ascontiguousarray(value, dtype=np.float64)
                assert first.shape == (self.V + 1,) and frame.shape == value.shape
                d = Events(first.ctypes.data, frame.ctypes.data, value.ctypes.data)
                keep += [first, frame, value]
                arrs.append(d)
                continue
            if ty == "bits":                 # [nframes][V] of 0 / 1 -> uint32 words [nframes][(V + 31) / 32], voice v = bit v % 32 of word v / 32
                a = pack_bits(inputs[n])
                assert a.shape == (nframes, (self.V + 31) // 32)
            else:
                a = np.ascontiguousarray(inputs[n], dtype=np.uint8 if ty == "u8" else np.float64)
                assert a.shape == (nframes, self.V)
            arrs.append(a)
        ptrs = (C.c_void_p * max(1, len(arrs)))(*[C.addressof(a) if isinstance(a, Events) else a.ctypes.data for a in arrs])
        out = np.empty((nframes, self.V), dtype=np.float64) if want_out else None
        mix = np.empty((nframes, 2), dtype=np.float64) if want_mix else None
        check(lib().mxb_patch_process(self.h, nframes, ptrs, _np_ptr(out), _np_ptr(mix), MEM_HOST, None), "mxb_patch_process")
        return out, mix
