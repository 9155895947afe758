"""ctypes loader for the two CPU oracles -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this module (see oracle/oracle_api.h).  The product package
maximilian_b200 never does.

    load("port")       oracle/libmaxioracle.so   (oracle/maxi_oracle.c, plain-C restatement)
    load("reference")  oracle/_ref/libmaxiref.so (the unmodified reference, compiled from a
                       checkout of it by oracle/Makefile; absent if never built)
"""
import ctypes as C
import os
import subprocess
import threading

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PATHS = {"port": os.path.join(HERE, "libmaxioracle.so"),
         "reference": os.path.join(HERE, "_ref", "libmaxiref.so"),
         # the same unmodified sources at -O3 -march=x86-64-v3: a CPU baseline to TIME (bench.py), never a checker
         "reference_o3": os.path.join(HERE, "_ref", "libmaxiref_o3.so")}

# stage selectors / ids: keep in sync with oracle_api.h
OSC = dict(sinewave=0, coswave=1, phasor=2, saw=3, square=4, pulse=5, impulse=6, triangle=7, phasorbetween=8)
FILT = dict(none=0, lores=1, hires=2, svf=3, biquad=4)
BIQUAD = dict(lowpass=0, highpass=1, bandpass=2, notch=3, peak=4, lowshelf=5, highshelf=6)
P = dict(freq=0, phase=1, duty=2, cutoff=3, resonance=4, gain=5, env_attack=6, env_decay=7,
         env_sustain=8, env_release=9, env_holdtime=10, delay_size=11, delay_feedback=12, pan=13, delay_position=14,
         phasor_start=15, phasor_end=16, filt0=32, filt1=33, filt2=34, env_amplitude=35, env_output=36, env_holdcount=37,
         env_flags=38, delay_phase=39, osc_output=40)


ENV_KIND = {False: 0, None: 0, True: 1, "adsr": 1, "ar": 2}
DELAY_KIND = {False: 0, None: 0, True: 1, "dl": 1, "position": 2}


class Chain(C.Structure):
    _fields_ = [("sample_rate", C.c_int32), ("osc_kind", C.c_int32), ("filt_kind", C.c_int32),
                ("biquad_type", C.c_int32), ("env_kind", C.c_int32), ("delay_on", C.c_int32),
                ("delay_capacity", C.c_int32), ("reserved", C.c_int32), ("svf_mix", C.c_double * 4)]


def build(kind="port"):
    """Compile the oracle library with oracle/Makefile (building the checker is not using it)."""
    target = "port" if kind == "port" else "ref"
    subprocess.check_call(["make", "-s", "-C", HERE, target])


_libs = {}


def available(kind):
    return os.path.exists(PATHS[kind])


def load(kind="port"):
    if kind in _libs:
        return _libs[kind]
    path = PATHS[kind]
    if not os.path.exists(path):
        build(kind)
    lib = C.CDLL(path)
    dp, ip, fp, vp = C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_float), C.c_void_p
    i32 = C.c_int32
    sig = {
        "mxo_kind": (C.c_char_p, []),
        "mxo_bank_create": (vp, [C.POINTER(Chain), i32]),
        "mxo_bank_destroy": (None, [vp]),
        "mxo_bank_set": (i32, [vp, i32, dp]),
        "mxo_bank_get": (i32, [vp, i32, dp]),
        "mxo_bank_process": (i32, [vp, i32, ip, ip, dp, dp, i32, i32]),
        "mxo_bank_process_fm": (i32, [vp, i32, dp, ip, ip, dp, dp, i32, i32]),
        "mxo_bank_process_mod": (i32, [vp, i32, dp, dp, dp, ip, ip, dp, dp, i32, i32]),
        "mxo_bank_process_mod2": (i32, [vp, i32, dp, dp, dp, C.POINTER(C.c_uint8), ip, ip, dp, dp, i32, i32]),
        "mxo_bank_get_ring": (i32, [vp, i32, dp, i32]),
        "mxo_env_attack_coeff": (C.c_double, [C.c_double, i32]),
        "mxo_env_attack_ms_coeff": (C.c_double, [C.c_double, i32]),
        "mxo_env_decay_coeff": (C.c_double, [C.c_double, i32]),
        "mxo_stft_create": (vp, [i32, i32, i32]),
        "mxo_stft_destroy": (None, [vp]),
        "mxo_stft_process": (i32, [vp, fp, i32, i32, fp, fp, fp, fp]),
        "mxo_stft_window": (i32, [vp, fp]),
        "mxo_spectral_features": (i32, [fp, i32, i32, i32, fp, fp, fp]),
        "mxo_mfcc_create": (vp, [i32, i32, i32, C.c_double, C.c_double, i32]),
        "mxo_mfcc_destroy": (None, [vp]),
        "mxo_mfcc_process": (i32, [vp, fp, i32, dp, dp]),
        "mxo_istft_create": (vp, [i32, i32, i32]),
        "mxo_istft_destroy": (None, [vp]),
        "mxo_istft_process": (i32, [vp, fp, fp, i32, fp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = res, args
    assert kind.startswith(lib.mxo_kind().decode()), (lib.mxo_kind(), kind)
    _libs[kind] = lib
    return lib


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double)) if a is not None else None


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float)) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32)) if a is not None else None


class Bank:
    """V voices of  osc -> [adsr] -> [filter] -> [delay] -> out / stereo mix  on the CPU."""

    def __init__(self, voices, osc="saw", filt="none", env=False, delay=False, sample_rate=48000,
                 biquad_type="lowpass", svf_mix=(1.0, 0.0, 0.0, 0.0), delay_capacity=4096, kind="port"):
        self.lib = load(kind)
        self.V = int(voices)
        # env: False | True/"adsr" | "ar";  delay: False | True/"dl" | "position" (dlFromPosition)
        ch = Chain(sample_rate, OSC[osc], FILT[filt], BIQUAD[biquad_type], ENV_KIND[env],
                   DELAY_KIND[delay], delay_capacity, 0, (C.c_double * 4)(*svf_mix))
        self.h = self.lib.mxo_bank_create(C.byref(ch), self.V)
        if not self.h:
            raise RuntimeError("mxo_bank_create failed")

    def close(self):
        if self.h:
            self.lib.mxo_bank_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set(self, name, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        rc = self.lib.mxo_bank_set(self.h, P[name], _dp(a))
        if rc:
            raise RuntimeError(f"mxo_bank_set({name}) -> {rc}")

    def get(self, name):
        a = np.empty(self.V, dtype=np.float64)
        rc = self.lib.mxo_bank_get(self.h, P[name], _dp(a))
        if rc:
            raise RuntimeError(f"mxo_bank_get({name}) -> {rc}")
        return a

    def ring(self, v, n):
        a = np.empty(n, dtype=np.float64)
        rc = self.lib.mxo_bank_get_ring(self.h, v, _dp(a), n)
        if rc:
            raise RuntimeError(f"mxo_bank_get_ring -> {rc}")
        return a

    def process(self, nframes, trig_on=None, trig_off=None, want_out=True, want_mix=False, threads=1, out=None, freq_tv=None,
                cutoff_tv=None, delay_size_tv=None, trig_tv=None):
        """Returns (out[nframes][V] or None, mix[nframes][2] or None). `out` may be a preallocated buffer.
        freq_tv / cutoff_tv / delay_size_tv: optional per-sample oscillator frequency / filter cutoff / delay size [nframes][V]."""
        if want_out and out is None:
            out = np.empty((nframes, self.V), dtype=np.float64)
        if not want_out:
            out = None
        if trig_tv is not None:
            tv = np.ascontiguousarray(trig_tv, dtype=np.uint8)
            assert tv.shape == (nframes, self.V) and trig_on is None
            f = np.ascontiguousarray(freq_tv, dtype=np.float64) if freq_tv is not None else None
            cu = np.ascontiguousarray(cutoff_tv, dtype=np.float64) if cutoff_tv is not None else None
            ds = np.ascontiguousarray(delay_size_tv, dtype=np.float64) if delay_size_tv is not None else None
            assert ds is None or ds.shape == (nframes, self.V)
            mix = np.empty((nframes, 2), dtype=np.float64) if want_mix else None
            rc = self.lib.mxo_bank_process_mod2(self.h, nframes, _dp(f), _dp(cu), _dp(ds), tv.ctypes.data_as(C.POINTER(C.c_uint8)), None, None,
                                                _dp(out), _dp(mix), 0, self.V)
            if rc:
                raise RuntimeError(f"mxo_bank_process_mod2 -> {rc}")
            return out, mix
        if freq_tv is not None or cutoff_tv is not None or delay_size_tv is not None:
            f = np.ascontiguousarray(freq_tv, dtype=np.float64) if freq_tv is not None else None
            cu = np.ascontiguousarray(cutoff_tv, dtype=np.float64) if cutoff_tv is not None else None
            ds = np.ascontiguousarray(delay_size_tv, dtype=np.float64) if delay_size_tv is not None else None
            assert ds is None or ds.shape == (nframes, self.V)
            assert f is None or f.shape == (nframes, self.V)
            assert cu is None or cu.shape == (nframes, self.V)
            ton = np.ascontiguousarray(trig_on, dtype=np.int32) if trig_on is not None else None
            toff = np.ascontiguousarray(trig_off, dtype=np.int32) if trig_off is not None else None
            mix = np.empty((nframes, 2), dtype=np.float64) if want_mix else None
            rc = self.lib.mxo_bank_process_mod(self.h, nframes, _dp(f), _dp(cu), _dp(ds), _ip(ton), _ip(toff), _dp(out), _dp(mix), 0, self.V)
            if rc:
                raise RuntimeError(f"mxo_bank_process_mod -> {rc}")
            return out, mix
        ton = np.ascontiguousarray(trig_on, dtype=np.int32) if trig_on is not None else None
        toff = np.ascontiguousarray(trig_off, dtype=np.int32) if trig_off is not None else None
        threads = max(1, min(int(threads), self.V))
        if threads == 1:
            mix = np.empty((nframes, 2), dtype=np.float64) if want_mix else None
            rc = self.lib.mxo_bank_process(self.h, nframes, _ip(ton), _ip(toff), _dp(out), _dp(mix), 0, self.V)
            if rc:
                raise RuntimeError(f"mxo_bank_process -> {rc}")
            return out, mix
        # voices statically partitioned over host threads (ctypes drops the GIL inside the call)
        bounds = np.linspace(0, self.V, threads + 1).astype(int)
        mixes = [np.empty((nframes, 2), dtype=np.float64) if want_mix else None for _ in range(threads)]
        rcs = [0] * threads

        def work(i):
            rcs[i] = self.lib.mxo_bank_process(self.h, nframes, _ip(ton), _ip(toff), _dp(out), _dp(mixes[i]),
                                               int(bounds[i]), int(bounds[i + 1] - bounds[i]))
        ts = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
        [t.start() for t in ts]
        [t.join() for t in ts]
        if any(rcs):
            raise RuntimeError(f"mxo_bank_process -> {rcs}")
        mix = None
        if want_mix:
            mix = mixes[0].copy()
            for m in mixes[1:]:
                mix += m
        return out, mix


def run_blocks_threaded(bank, nframes, gates, threads, out):
    """CPU-baseline driver: `len(gates)` consecutive blocks, voices statically partitioned over `threads` host
    threads; every thread runs ALL blocks of its own voices (voices are independent, so no barrier between
    blocks) -- one thread start per run, the time goes to the reference's per-sample loops.
    gates: list of (trig_on, trig_off) int32 arrays or (None, None); out: [nframes][V] float64, reused."""
    threads = max(1, min(int(threads), bank.V))
    bounds = np.linspace(0, bank.V, threads + 1).astype(int)
    rcs = [0] * threads

    def work(i):
        lo, n = int(bounds[i]), int(bounds[i + 1] - bounds[i])
        for on, off in gates:
            rc = bank.lib.mxo_bank_process(bank.h, nframes, _ip(on), _ip(off), _dp(out), None, lo, n)
            if rc:
                rcs[i] = rc
                return
    ts = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
    [t.start() for t in ts]
    [t.join() for t in ts]
    if any(rcs):
        raise RuntimeError(f"mxo_bank_process -> {rcs}")


class Stft:
    def __init__(self, channels, fft_size=1024, hop=512, kind="port"):
        self.lib = load(kind)
        self.C, self.n, self.hop, self.bins = channels, fft_size, hop, fft_size // 2
        self.h = self.lib.mxo_stft_create(channels, fft_size, hop)
        if not self.h:
            raise RuntimeError("mxo_stft_create failed")

    def __del__(self):
        try:
            if self.h:
                self.lib.mxo_stft_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def window(self):
        w = np.empty(self.n, dtype=np.float32)
        self.lib.mxo_stft_window(self.h, _fp(w))
        return w

    def process(self, x, want=("mags", "phases", "re", "im")):
        """x: float32 [C][n] planar. Returns dict of float32 [C][frames][bins]."""
        x = np.ascontiguousarray(x, dtype=np.float32)
        assert x.shape[0] == self.C
        n = x.shape[1]
        maxf = n // self.hop + 2
        bufs = {k: (np.zeros((self.C, maxf, self.bins), dtype=np.float32) if k in want else None)
                for k in ("mags", "phases", "re", "im")}
        f = self.lib.mxo_stft_process(self.h, _fp(x), n, maxf, _fp(bufs["mags"]), _fp(bufs["phases"]),
                                      _fp(bufs["re"]), _fp(bufs["im"]))
        if f < 0:
            raise RuntimeError(f"mxo_stft_process -> {f}")
        return {k: np.ascontiguousarray(v[:, :f]) for k, v in bufs.items() if v is not None}


def spectral_features(mags, fft_size, sample_rate=48000, kind="port"):
    """mags float32 [..., bins] -> (db [..., bins], flatness [...], centroid [...]) : maxiFFT::magsToDB / spectralFlatness / spectralCentroid."""
    lib = load(kind)
    m = np.ascontiguousarray(mags, dtype=np.float32)
    lead = m.shape[:-1]
    n = int(np.prod(lead)) if lead else 1
    db = np.empty_like(m); fl = np.empty(n, dtype=np.float32); ce = np.empty(n, dtype=np.float32)
    rc = lib.mxo_spectral_features(_fp(m), n, fft_size, sample_rate, _fp(db), _fp(fl), _fp(ce))
    if rc:
        raise RuntimeError(f"mxo_spectral_features -> {rc}")
    return db, fl.reshape(lead), ce.reshape(lead)


class Mfcc:
    def __init__(self, num_bins=512, num_filters=42, num_coeffs=40, min_freq=20.0, max_freq=20000.0,
                 sample_rate=48000, kind="port"):
        self.lib = load(kind)
        self.bins, self.filters, self.coeffs = num_bins, num_filters, num_coeffs
        self.h = self.lib.mxo_mfcc_create(num_bins, num_filters, num_coeffs, min_freq, max_freq, sample_rate)
        if not self.h:
            raise RuntimeError("mxo_mfcc_create failed")

    def __del__(self):
        try:
            if self.h:
                self.lib.mxo_mfcc_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def process(self, mags):
        """mags float32 [..., bins] -> (coeffs [..., numCoeffs], melbands [..., numFilters])."""
        m = np.ascontiguousarray(mags, dtype=np.float32)
        lead = m.shape[:-1]
        n = int(np.prod(lead)) if lead else 1
        co = np.empty((n, self.coeffs), dtype=np.float64)
        mb = np.empty((n, self.filters), dtype=np.float64)
        rc = self.lib.mxo_mfcc_process(self.h, _fp(m), n, _dp(co), _dp(mb))
        if rc:
            raise RuntimeError(f"mxo_mfcc_process -> {rc}")
        return co.reshape(lead + (self.coeffs,)), mb.reshape(lead + (self.filters,))


class Istft:
    def __init__(self, channels, fft_size=1024, hop=512, kind="port"):
        self.lib = load(kind)
        self.C, self.n, self.hop, self.bins = channels, fft_size, hop, fft_size // 2
        self.h = self.lib.mxo_istft_create(channels, fft_size, hop)
        if not self.h:
            raise RuntimeError("mxo_istft_create failed")

    def __del__(self):
        try:
            if self.h:
                self.lib.mxo_istft_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def process(self, mags, phases):
        """mags/phases float32 [C][frames][bins] -> float32 [C][frames*hop]."""
        m = np.ascontiguousarray(mags, dtype=np.float32)
        p = np.ascontiguousarray(phases, dtype=np.float32)
        frames = m.shape[1]
        out = np.empty((self.C, frames * self.hop), dtype=np.float32)
        rc = self.lib.mxo_istft_process(self.h, _fp(m), _fp(p), frames, _fp(out))
        if rc:
            raise RuntimeError(f"mxo_istft_process -> {rc}")
        return out


# ------------------------------------------------------------------------------------------------ voice patches

class MxoStage(C.Structure):
    _fields_ = [("op", C.c_int32), ("kind", C.c_int32), ("dst", C.c_int32), ("reserved", C.c_int32), ("src", C.c_int32 * 8)]


class MxoEnvgenShape(C.Structure):
    _fields_ = [("stages", C.c_int32), ("loop", C.c_int32), ("retrigger", C.c_int32),
                ("levels", C.POINTER(C.c_double)), ("times", C.POINTER(C.c_double)), ("curves", C.POINTER(C.c_double))]


class MxoPatchDesc(C.Structure):
    _fields_ = [("voices", C.c_int32), ("n_stages", C.c_int32), ("n_params", C.c_int32), ("n_consts", C.c_int32), ("n_inputs", C.c_int32),
                ("sample_rate", C.c_int32), ("delay_taps", C.c_int32), ("n_shapes", C.c_int32),
                ("stages", C.POINTER(MxoStage)), ("consts", C.POINTER(C.c_double)), ("shapes", C.POINTER(MxoEnvgenShape))]


def _doubles(x):
    return (C.c_double * max(1, len(x)))(*x)


def _patch_sigs(lib):
    if getattr(lib, "_patch_sigs_done", False):
        return
    dp, vp, i32 = C.POINTER(C.c_double), C.c_void_p, C.c_int32
    lib.mxo_set_tables.restype, lib.mxo_set_tables.argtypes = i32, [dp, dp, C.c_double]
    lib.mxo_get_tables.restype, lib.mxo_get_tables.argtypes = i32, [dp, dp, dp]
    lib.mxo_patch_create.restype, lib.mxo_patch_create.argtypes = vp, [C.POINTER(MxoPatchDesc)]
    lib.mxo_patch_destroy.restype, lib.mxo_patch_destroy.argtypes = None, [vp]
    lib.mxo_patch_set_param.restype, lib.mxo_patch_set_param.argtypes = i32, [vp, i32, dp]
    lib.mxo_patch_set_state.restype, lib.mxo_patch_set_state.argtypes = i32, [vp, i32, i32, dp]
    lib.mxo_patch_get_state.restype, lib.mxo_patch_get_state.argtypes = i32, [vp, i32, i32, dp]
    lib.mxo_patch_get_ring.restype, lib.mxo_patch_get_ring.argtypes = i32, [vp, i32, i32, dp, i32]
    lib.mxo_patch_process.restype, lib.mxo_patch_process.argtypes = i32, [vp, i32, C.POINTER(C.c_void_p), dp, dp]
    lib.mxo_noise_fill.restype, lib.mxo_noise_fill.argtypes = None, [C.c_uint32, C.c_int64, dp]
    lib.mxo_srand.restype, lib.mxo_srand.argtypes = None, [C.c_uint32]
    lib._patch_sigs_done = True


def noise_fill(seed, n, kind="port"):
    """srand(seed), then n values of maxiOsc::noise() (src/maximilian.cpp:214-220) from this process's libc rand()."""
    lib = load(kind); _patch_sigs(lib)
    a = np.empty(int(n), dtype=np.float64)
    lib.mxo_noise_fill(int(seed), int(n), _dp(a))
    return a


def srand(seed, kind="reference"):
    """Re-seed libc rand() (process-wide) before the compiled reference runs a patch whose chorus stage draws from it."""
    lib = load(kind); _patch_sigs(lib)
    lib.mxo_srand(int(seed))


def get_tables(kind="reference"):
    """(sineBuffer[514], transition[1001], sine_before) as the library `kind` holds them (the compiled reference: its own)."""
    lib = load(kind); _patch_sigs(lib)
    s = np.empty(514); t = np.empty(1001); b = C.c_double(0.0)
    rc = lib.mxo_get_tables(_dp(s), _dp(t), C.byref(b))
    if rc:
        raise RuntimeError(f"mxo_get_tables -> {rc}")
    return s, t, b.value


def per_sample_roundtrip(x, fft_size, hop, kind="reference"):
    """The compiled reference's maxiFFT + maxiIFFT called once per sample (ref_shim: mxo_ref_per_sample_roundtrip) on one channel x[1][N]:
    (frames fired, resynthesised y[N] fp32, fired[N] uint8 -- 1 where fft.process returned true)."""
    lib = load(kind)
    fn = lib.mxo_ref_per_sample_roundtrip
    fn.restype = C.c_int32
    fn.argtypes = [C.POINTER(C.c_float), C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_float), C.POINTER(C.c_uint8)]
    x = np.ascontiguousarray(x, dtype=np.float32)
    N = x.shape[-1]
    y = np.empty(N, dtype=np.float32); fired = np.empty(N, dtype=np.uint8)
    F = fn(_fp(x), N, fft_size, hop, _fp(y), fired.ctypes.data_as(C.POINTER(C.c_uint8)))
    return int(F), y, fired


def set_tables(sine514, transition1001, sine_before, kind="port"):
    lib = load(kind); _patch_sigs(lib)
    s = np.ascontiguousarray(sine514, dtype=np.float64); t = np.ascontiguousarray(transition1001, dtype=np.float64)
    rc = lib.mxo_set_tables(_dp(s), _dp(t), float(sine_before))
    if rc:
        raise RuntimeError(f"mxo_set_tables -> {rc}")


class Patch:
    """A maximilian_b200.patchdef.PatchDef on the CPU (kind: 'port' = maxi_oracle.c, 'reference' = the reference's own objects)."""

    def __init__(self, defn, voices, sample_rate=48000, delay_taps=0, kind="port", **_):
        self.lib = load(kind); _patch_sigs(self.lib)
        self.defn, self.V = defn, int(voices)
        st = (MxoStage * len(defn.stages))()
        for i, (op, k, dst, src) in enumerate(defn.stages):
            st[i].op, st[i].kind, st[i].dst, st[i].reserved = op, k, dst, 0
            for j in range(8):
                st[i].src[j] = src[j]
        consts = _doubles(defn.consts)
        shapes = (MxoEnvgenShape * max(1, len(defn.shapes)))()
        keep = [st, consts, shapes]
        for i, (lv, tm, cv, loop, retrig) in enumerate(defn.shapes):
            arrs = _doubles(lv), _doubles(tm), _doubles(cv)
            shapes[i] = MxoEnvgenShape(len(tm), int(loop), int(retrig), *arrs)
            keep += arrs
        d = MxoPatchDesc(self.V, len(defn.stages), len(defn.params), len(defn.consts), len(defn.inputs), sample_rate, int(delay_taps),
                         len(defn.shapes), st, consts, shapes)
        self._keep = keep
        self.h = self.lib.mxo_patch_create(C.byref(d))
        if not self.h:
            raise RuntimeError("mxo_patch_create failed")

    def __del__(self):
        try:
            if self.h:
                self.lib.mxo_patch_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def set(self, name, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        rc = self.lib.mxo_patch_set_param(self.h, self.defn.params.index(name), _dp(a))
        if rc:
            raise RuntimeError(f"mxo_patch_set_param({name}) -> {rc}")

    def get_state(self, stage, slot):
        a = np.empty(self.V, dtype=np.float64)
        rc = self.lib.mxo_patch_get_state(self.h, stage, slot, _dp(a))
        if rc:
            raise RuntimeError(f"mxo_patch_get_state -> {rc}")
        return a

    def set_state(self, stage, slot, values):
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(values, dtype=np.float64), (self.V,)))
        rc = self.lib.mxo_patch_set_state(self.h, stage, slot, _dp(a))
        if rc:
            raise RuntimeError(f"mxo_patch_set_state -> {rc}")

    def ring(self, stage, v, n):
        a = np.empty(n, dtype=np.float64)
        rc = self.lib.mxo_patch_get_ring(self.h, stage, v, _dp(a), n)
        if rc:
            raise RuntimeError(f"mxo_patch_get_ring -> {rc}")
        return a

    def process(self, nframes, inputs=None, want_out=True, want_mix=False):
        inputs = inputs or {}
        arrs = [np.ascontiguousarray(inputs[n], dtype=np.float64) for n in self.defn.inputs]
        for a in arrs:
            assert a.shape == (nframes, self.V)
        ptrs = (C.c_void_p * max(1, len(arrs)))(*[a.ctypes.data for a in arrs])
        out = np.empty((nframes, self.V), dtype=np.float64) if want_out else None
        mix = np.empty((nframes, 2), dtype=np.float64) if want_mix else None
        rc = self.lib.mxo_patch_process(self.h, nframes, ptrs, _dp(out), _dp(mix))
        if rc:
            raise RuntimeError(f"mxo_patch_process -> {rc}")
        return out, mix


# ------------------------------------------------------------------------------------------------ octave analyser / bark

def _post_sigs(lib):
    if getattr(lib, "_post_sigs_done", False):
        return
    fp, dp, vp, i32 = C.POINTER(C.c_float), C.POINTER(C.c_double), C.c_void_p, C.c_int32
    lib.mxo_octave_create.restype, lib.mxo_octave_create.argtypes = vp, [i32, C.c_float, i32, i32]
    lib.mxo_octave_destroy.restype, lib.mxo_octave_destroy.argtypes = None, [vp]
    lib.mxo_octave_n_averages.restype, lib.mxo_octave_n_averages.argtypes = i32, [vp]
    lib.mxo_octave_config.restype, lib.mxo_octave_config.argtypes = i32, [vp, i32, C.c_float, C.c_float, C.c_float]
    lib.mxo_octave_process.restype, lib.mxo_octave_process.argtypes = i32, [vp, fp, i32, fp, fp]
    lib.mxo_bark.restype, lib.mxo_bark.argtypes = i32, [fp, i32, i32, i32, dp, dp, dp]
    lib._post_sigs_done = True


class Octave:
    """maxiFFTOctaveAnalyzer per channel: mags float32 [C][frames][bands] -> (averages, peaks) float32 [C][frames][nAverages]."""

    def __init__(self, channels, sampling_rate, n_bands, n_per_octave, kind="port"):
        self.lib = load(kind); _post_sigs(self.lib)
        self.C, self.bands = channels, n_bands
        self.h = self.lib.mxo_octave_create(channels, float(sampling_rate), n_bands, n_per_octave)
        if not self.h:
            raise RuntimeError("mxo_octave_create failed")
        self.n_averages = self.lib.mxo_octave_n_averages(self.h)

    def __del__(self):
        try:
            if self.h:
                self.lib.mxo_octave_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def config(self, peak_hold_time=0, peak_decay_rate=0.9, eq_intercept=1.0, eq_slope=0.0):
        self.lib.mxo_octave_config(self.h, int(peak_hold_time), float(peak_decay_rate), float(eq_intercept), float(eq_slope))

    def process(self, mags):
        m = np.ascontiguousarray(mags, dtype=np.float32)
        assert m.shape[0] == self.C and m.shape[2] == self.bands
        f = m.shape[1]
        av = np.empty((self.C, f, self.n_averages), dtype=np.float32); pk = np.empty_like(av)
        rc = self.lib.mxo_octave_process(self.h, _fp(m), f, _fp(av), _fp(pk))
        if rc:
            raise RuntimeError(f"mxo_octave_process -> {rc}")
        return av, pk


def bark(spectrum, sample_rate, buffer_size, kind="port"):
    """maxiBark on float32 [..., buffer_size/2] -> (specific [..., 24], relative [..., 24], total [...])."""
    lib = load(kind); _post_sigs(lib)
    m = np.ascontiguousarray(spectrum, dtype=np.float32)
    lead = m.shape[:-1]
    n = int(np.prod(lead)) if lead else 1
    sp = np.empty((n, 24)); rl = np.empty((n, 24)); tt = np.empty(n)
    rc = lib.mxo_bark(_fp(m), n, int(sample_rate), int(buffer_size), _dp(sp), _dp(rl), _dp(tt))
    if rc:
        raise RuntimeError(f"mxo_bark -> {rc}")
    return sp.reshape(lead + (24,)), rl.reshape(lead + (24,)), tt.reshape(lead)
