/*
 * maximilian_b200.hpp -- C++ host layer over the C ABI (maxib200.h), keeping the reference's class surface:
 *   maxiSettings, maxiOsc, maxiFilter, maxiSVF, maxiBiquad, maxiEnv, maxiDelayline, maxiMix   (src/maximilian.h)
 *   maxiFFT, maxiIFFT, maxiMFCC                                                               (src/libs/maxiFFT.h, maxiMFCC.h)
 * with the same method names and argument meaning, restructured from "one call = one sample of one object"
 * to "one call = one BLOCK of a whole bank of voices":
 *
 *   reference patch (per sample, per voice)              this header (per block, V voices)
 *   ------------------------------------------------     -------------------------------------------------
 *   maxiOsc osc[V]; maxiSVF svf[V]; maxiMix mix;          maxiVoices voices(V);
 *                                                          maxiOsc osc(voices); maxiSVF svf(voices); maxiMix mix(voices);
 *   void play(double* out) {                              void play(maxiVoices& v) {
 *     for (i < V) {                                         maxiSignal w = svf.play(osc.saw(freq), 1, 0, 0, 0);
 *       w = svf[i].play(osc[i].saw(f[i]), 1,0,0,0);         mix.stereo(w, v.bus(), pan);
 *       mix.stereo(w, two, pan[i]); out[0] += two[0]...   }
 *   } }
 *   routing(): for each frame: play(frame)                maxiRouting(): play(voices) once, then one fused kernel
 *   (cpp/commandline/player.cpp:25-44)                    renders nBufferFrames frames of every voice
 *
 * The calls inside play() do not compute anything on the host: they describe the chain
 * (oscillator -> [maxiEnv::adsr] -> [filter] -> [maxiDelayline::dl] -> maxiMix::stereo / per-voice output) and hand
 * over per-voice parameters; maxiVoices::render() executes the block on the GPU through mxb_bank_process. Chains the
 * kernels do not implement are rejected with an exception, never emulated: there is no CPU path in here.
 *
 * Error behaviour: the reference has none (UB, or exit(1) in fft.cpp:67,131). Here every failure of the C ABI
 * surfaces as a maxiError (std::runtime_error) carrying mxb_last_error().
 */
#ifndef MAXIMILIAN_B200_HPP
#define MAXIMILIAN_B200_HPP

#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <initializer_list>
#include <string>
#include <utility>
#include <vector>

#include "maxib200.h"

/* Source compatibility with patches written against src/maximilian.h (SURVEY.md 8b): the reference header pulls
 * namespace std in (:54) and defines these (:55-67), and user patches rely on both (`vector<double>`, `cout`, PI). */
#ifndef MAXIMILIAN_B200_NO_STD_NAMESPACE
using namespace std;
#endif
#ifndef PI
#define PI 3.1415926535897932384626433832795
#endif
#ifndef TWOPI
#define TWOPI 6.283185307179586476925286766559
#endif
#ifndef CHEERP_EXPORT
#define CHEERP_EXPORT
#endif

struct maxiError : std::runtime_error {
    int code;
    maxiError(int c, const std::string& what) : std::runtime_error(what), code(c) {}
};

namespace maxib200_detail {
inline void check(int rc, const char* what) {
    if (rc != MXB_OK) throw maxiError(rc, std::string(what) + ": " + mxb_last_error());
}
}  // namespace maxib200_detail

/* maxiSettings, src/maximilian.h:117-163: process-global sample rate / channels / buffer size. */
class maxiSettings {
public:
    static inline size_t sampleRate = 44100;   /* defaults of src/maximilian.cpp:57-59 */
    static inline size_t channels = 2;
    static inline size_t bufferSize = 1024;
    static void setup(size_t initSampleRate, size_t initChannels, size_t initBufferSize) {
        sampleRate = initSampleRate; channels = initChannels; bufferSize = initBufferSize;
    }
    static size_t getSampleRate() { return sampleRate; }
};

/* A per-voice parameter: one double per voice (a std::vector that outlives play()), or a scalar (what the reference passes by
 * value on every sample). Scalars are compiled into the patch as constants: a scalar that changes from block to block is a
 * different patch -- pass a per-voice vector for block-rate control. */
class maxiParam {
public:
    maxiParam(double scalar = 0.0) : scalar_(scalar), vec_(nullptr) {}
    maxiParam(int scalar) : scalar_((double)scalar), vec_(nullptr) {}
    maxiParam(const std::vector<double>& perVoice) : scalar_(0.0), vec_(&perVoice) {}
    bool isScalar() const { return vec_ == nullptr; }
    double scalar() const { return scalar_; }
    const std::vector<double>& vec() const { return *vec_; }
private:
    double scalar_;
    const std::vector<double>* vec_;
};

/* trigger_v(t) == 1 for on[v] <= t < off[v], t counting frames inside the current block (a sample-accurate note gate) */
struct maxiGate {
    const std::vector<int32_t>* on = nullptr;
    const std::vector<int32_t>* off = nullptr;
    maxiGate() {}
    maxiGate(const std::vector<int32_t>& on_, const std::vector<int32_t>& off_) : on(&on_), off(&off_) {}
};
/* a per-sample control stream for the current block: values[t * voices + v] (maxiEnv::trigger written by the patch on any sample,
 * audio-rate modulation computed elsewhere) */
struct maxiStream {
    const double* values = nullptr;
    explicit maxiStream(const double* v) : values(v) {}
    explicit maxiStream(const std::vector<double>& v) : values(v.data()) {}
};

class maxiVoices;
/* Control events of the current block, for one value of every voice: the reference's play() writes members such as currentPitch or
 * ADSR[voice].trigger on some samples, and the value holds until the next write. The control code calls set(frame, voice, value) during the
 * block; render() hands the events over as an MXB_IN_EVENTS stream -- per voice, in call order -- and clears them. The stream reads each
 * voice's held value: it starts at 0.0 and carries over from block to block (mxb_patch_get_held / set_held on patchHandle()). For a list
 * in frame order that is the value of the last event at or before the sample; an event at a negative frame applies at frame 0, one at
 * frame >= nFrames is dropped with every later one of that voice. It costs 16 bytes per event, where a maxiStream costs 8 per voice-sample.
 * Usable wherever a maxiStream is, and as any stage argument (maxiArg).
 * A one-sample trigger (the reference sets `trigger = 1` on a tick and back to 0 after that sample) is two events: set(t, v, 1) and
 * set(t + 1, v, 0); when t is the block's last frame, the second belongs at frame 0 of the next block. */
class maxiEvents {
public:
    explicit maxiEvents(maxiVoices& v);
    void set(int frame, int voice, double value) {
        if (voice < 0 || voice >= V_) throw maxiError(MXB_ERR_INVALID, "maxiEvents::set: voice " + std::to_string(voice) + " of " + std::to_string(V_));
        ev_.push_back(Ev{voice, frame, value});
    }
private:
    friend class maxiVoices;
    struct Ev { int32_t voice, frame; double value; };
    /* the events of this block as a CSR list by voice (a stable counting sort: each voice keeps its call order); then cleared */
    const mxb_events* pack() {
        first_.assign((size_t)V_ + 1, 0);
        for (const Ev& e : ev_) first_[(size_t)e.voice + 1] += 1;
        for (int v = 0; v < V_; ++v) first_[(size_t)v + 1] += first_[(size_t)v];
        frame_.resize(ev_.size()); value_.resize(ev_.size());
        std::vector<int32_t> at(first_.begin(), first_.end() - 1);
        for (const Ev& e : ev_) { const size_t i = (size_t)at[(size_t)e.voice]++; frame_[i] = e.frame; value_[i] = e.value; }
        ev_.clear();
        desc_.first = first_.data(); desc_.frame = frame_.data(); desc_.value = value_.data();
        return &desc_;
    }
    maxiVoices* v_;
    int V_;
    std::vector<Ev> ev_;
    std::vector<int32_t> first_, frame_;
    std::vector<double> value_;
    mxb_events desc_{};
};

/* The signal flowing between the calls of a play(): a handle to a value of the recorded program (register, parameter or constant). */
struct maxiSignal {
    maxiVoices* voices = nullptr;
    int32_t src = MXB_NONE;
    int stage = 0;                      /* 1 osc, 2 env, 3 filter, 4 delay, 0 anything else */
};
struct maxiBus { maxiVoices* voices = nullptr; };

/* The voices behind one play(). The calls made inside play() do not compute anything on the host: they RECORD the patch -- a
 * stage per call, `+ - * /` between signals included -- and hand over parameters; render() runs the block on the GPU. A patch of the
 * shape oscillator -> [maxiEnv] -> [filter] -> [maxiDelayline] -> maxiMix::stereo / per-voice output with block-constant arguments
 * runs on the fused bank kernels (mxb_bank, the HBM-roofline path); any other graph -- sums of oscillators, an LFO on a cutoff,
 * the envelope applied after the filter (maximilian_examples/15.polysynth/main.cpp:54-70), per-sample triggers -- runs as a voice
 * patch (mxb_patch: a kernel generated and compiled for the recorded graph, or the interpreting kernel). The patch must be the same on
 * every block (the reference's play() is, too). */
class maxiVoices {
public:
    explicit maxiVoices(int voices, int device = 0) : V_(voices), device_(device) {}
    ~maxiVoices() { if (bank_) mxb_bank_destroy(bank_); if (patch_) mxb_patch_destroy(patch_); if (ctx_) mxb_ctx_destroy(ctx_); }
    maxiVoices(const maxiVoices&) = delete;
    maxiVoices& operator=(const maxiVoices&) = delete;

    int size() const { return V_; }
    maxiBus bus() { return maxiBus{this}; }
    /* sineBuffer / transition of the reference (src/maximilian.cpp:63, 67) for sinebuf / sinebuf4 / sawn: see mxb_ctx_set_tables */
    void setTables(const double* sine514, const double* transition1001, double sineBefore) {
        sine_.assign(sine514, sine514 + 514); trans_.assign(transition1001, transition1001 + 1001); sineBefore_ = sineBefore; haveTables_ = true;
    }
    /* ring slots per voice for maxiDelayline / maxiFlanger stages of an interpreted patch (a fused chain takes it from the object) */
    void setDelayCapacity(int taps) { taps_ = taps; }
    /* the sum over voices of `x` goes to bus channel 0 (what `mix += x` does in a reference play()) */
    void sum(maxiSignal x) { check(x, "maxiVoices::sum"); emit(MXB_OP_MIX_STEREO, 0, {x.src, constOp(0.0)}, false); }
    /* per-voice output: out[t][v] = x */
    void out(maxiSignal x) { check(x, "maxiVoices::out"); emit(MXB_OP_OUT, 0, {x.src}, false); outSrc_ = x.src; }

    /* Run the patch recorded since the last render for nFrames frames.
     * out:  per-voice samples [nFrames][V] (host memory) or nullptr (the last signal of the chain unless out() named one);
     * mix:  stereo bus [nFrames][2] (host memory, interleaved like RTAUDIO_FLOAT64) or nullptr. */
    void render(int nFrames, double* out, double* mix) {
        using maxib200_detail::check;
        if (prog_.empty()) throw maxiError(MXB_ERR_STATE, "maxiVoices::render: play() described nothing");
        if (!ctx_) check(mxb_ctx_create(device_, (int32_t)maxiSettings::sampleRate, &ctx_), "mxb_ctx_create");
        if (outSrc_ == MXB_NONE && lastSrc_ != MXB_NONE) { emit(MXB_OP_OUT, 0, {lastSrc_}, false); outSrc_ = lastSrc_; }   /* the chain's last signal */
        wantMix_ = false;
        for (const mxb_stage& g : prog_) wantMix_ = wantMix_ || g.op == MXB_OP_MIX_STEREO;
        if (!bank_ && !patch_) build(nFrames);
        else if (!sameProgram()) throw maxiError(MXB_ERR_UNSUPPORTED, "maxiVoices: play() recorded a different patch than on the first block");
        if (bank_) runBank(nFrames, out, mix); else runPatch(nFrames, out, mix);
        prog_.clear(); consts_.clear(); nParams_ = 0; nInputs_ = 0; nextReg_ = 0; gate_ = maxiGate(); gateInput_ = -1; outSrc_ = MXB_NONE; lastSrc_ = MXB_NONE;
        pendingPhase_.clear(); egObjs_.clear(); egShapes_.clear();
    }

    /* state read-back of a fused chain (checkpointing / tests): MXB_P_PHASE, MXB_S_* */
    std::vector<double> state(int id) {
        if (!bank_) throw maxiError(MXB_ERR_STATE, "maxiVoices::state: the graph runs as a voice patch (use patchHandle())");
        std::vector<double> v((size_t)V_);
        maxib200_detail::check(mxb_bank_get_state(bank_, id, v.data(), MXB_MEM_HOST), "mxb_bank_get_state");
        return v;
    }
    mxb_bank* handle() { return bank_; }
    mxb_patch* patchHandle() { return patch_; }
    bool fused() const { return bank_ != nullptr; }

    /* ---- recording interface (used by the maxi* classes and the operators below) ---- */
    int32_t constOp(double v) {
        for (size_t i = 0; i < consts_.size(); ++i) if (std::memcmp(&consts_[i], &v, sizeof(double)) == 0) return MXB_CONST((int32_t)i);
        consts_.push_back(v);
        return MXB_CONST((int32_t)consts_.size() - 1);
    }
    int32_t operand(const maxiParam& p) {
        if (p.isScalar()) return constOp(p.scalar());
        if (p.vec().size() != (size_t)V_) throw maxiError(MXB_ERR_INVALID, "maxiParam: per-voice vector has the wrong length");
        if ((size_t)nParams_ >= paramVals_.size()) { paramVals_.emplace_back(); paramDirty_.push_back(true); }
        std::vector<double>& dst = paramVals_[(size_t)nParams_];
        if (dst.size() != (size_t)V_ || std::memcmp(dst.data(), p.vec().data(), sizeof(double) * (size_t)V_) != 0) { dst = p.vec(); paramDirty_[(size_t)nParams_] = true; }
        return MXB_PARAM(nParams_++);
    }
    int32_t operand(const maxiSignal& x) { check(x, "operand"); return x.src; }
    int32_t operand(const maxiStream& st) { return input(st.values, MXB_IN_F64, nullptr); }
    int32_t operand(const maxiGate& g) {          /* an interval gate: a trigger stream built at render time (or the bank's own gate) */
        gate_ = g;
        gateInput_ = nInputs_;
        return input(nullptr, MXB_IN_F64, nullptr);
    }
    int32_t operand(const maxiEvents& ev) {       /* one events stream per maxiEvents object and block, however often it is read */
        if (ev.v_ != this) throw maxiError(MXB_ERR_UNSUPPORTED, "maxiEvents: the events belong to another maxiVoices");
        for (int k = 0; k < nInputs_; ++k) if (inputEv_[(size_t)k] == &ev) return MXB_INPUT(k);
        return input(nullptr, MXB_IN_EVENTS, const_cast<maxiEvents*>(&ev));
    }
    /* a stream or events as a signal of play(), for the arithmetic between the calls (`currentPitch * 0.5`): no stage of its own */
    maxiSignal signal(const maxiStream& st) { return maxiSignal{this, operand(st), 0}; }
    maxiSignal signal(const maxiEvents& ev) { return maxiSignal{this, operand(ev), 0}; }
    maxiSignal emit(int32_t op, int32_t kind, std::initializer_list<int32_t> srcs, bool wantDst = true, int stageTag = 0) {
        mxb_stage g;
        g.op = op; g.kind = kind; g.reserved = 0; g.dst = MXB_NONE;
        int k = 0;
        for (int32_t x : srcs) g.src[k++] = x;
        for (; k < MXB_STAGE_SRCS; ++k) g.src[k] = MXB_NONE;
        if (wantDst) {
            if (nextReg_ >= 16) throw maxiError(MXB_ERR_UNSUPPORTED, "maxiVoices: more than 16 values in one play()");
            g.dst = MXB_REG(nextReg_++);
        }
        prog_.push_back(g);
        if (wantDst) lastSrc_ = g.dst;
        return maxiSignal{this, g.dst, stageTag};
    }
    void check(const maxiSignal& x, const char* who) const {
        if (x.voices != this) throw maxiError(MXB_ERR_UNSUPPORTED, std::string(who) + ": the signal belongs to another maxiVoices");
    }
    int delayCapacity_ = 0;             /* of the maxiDelayline object of a fused chain */
    int biquadType_ = 0;

private:
    static bool blockConstant(int32_t s) { return s == MXB_NONE || (s >> 8) == 1 || (s >> 8) == 2; }   /* parameter or constant */
    int32_t input(const double* values, int32_t type, maxiEvents* ev) {
        if ((size_t)nInputs_ >= inputPtr_.size()) { inputPtr_.push_back(nullptr); inputType_.push_back(MXB_IN_F64); inputEv_.push_back(nullptr); }
        inputPtr_[(size_t)nInputs_] = values; inputType_[(size_t)nInputs_] = type; inputEv_[(size_t)nInputs_] = ev;
        return MXB_INPUT(nInputs_++);
    }
    bool sameProgram() const {
        return built_.size() == prog_.size() && std::memcmp(built_.data(), prog_.data(), sizeof(mxb_stage) * prog_.size()) == 0 &&
               builtConsts_.size() == consts_.size() && std::memcmp(builtConsts_.data(), consts_.data(), sizeof(double) * consts_.size()) == 0 &&
               builtShapes_ == egShapes_ && std::vector<int32_t>(inputType_.begin(), inputType_.begin() + nInputs_) == builtTypes_;
    }
    /* the shape of one maxiEnvGen object (maxiEnvGen::setup, setLoop, setRetrigger) */
    struct EgShape {
        std::vector<double> levels, times, curves;
        int loop = 0, retrigger = 0;
        bool operator==(const EgShape& o) const { return levels == o.levels && times == o.times && curves == o.curves && loop == o.loop && retrigger == o.retrigger; }
    };
    /* the shape index of a maxiEnvGen object in this block: objects are numbered in the order they first play */
    int32_t egShape(const void* obj, const EgShape& s) {
        for (size_t i = 0; i < egObjs_.size(); ++i) if (egObjs_[i] == obj) return (int32_t)i;
        egObjs_.push_back(obj); egShapes_.push_back(s);
        return (int32_t)egObjs_.size() - 1;
    }
    std::vector<double> values(int32_t s) const {       /* a block-constant operand as a per-voice array */
        if ((s >> 8) == 1) return paramVals_[(size_t)(s & 0xff)];
        return std::vector<double>((size_t)V_, s == MXB_NONE ? 0.0 : consts_[(size_t)(s & 0xff)]);
    }

    /* Does the recorded program have the shape of the fused kernels? osc -> [env(interval gate)] -> [filter] -> [delay] -> stereo / out,
     * every argument block-constant. Fills chain_ (which stage plays which role). */
    struct Chain { int osc = -1, env = -1, filt = -1, dly = -1, mix = -1, out = -1; };
    bool matchChain(Chain& c) const {
        size_t i = 0;
        const size_t n = prog_.size();
        auto args_const = [&](const mxb_stage& g, int from) { for (int k = from; k < MXB_STAGE_SRCS; ++k) if (!blockConstant(g.src[k])) return false; return true; };
        if (i >= n || prog_[i].op != MXB_OP_OSC || prog_[i].kind > MXB_OSC_PHASORBETWEEN || !args_const(prog_[i], 0)) return false;
        c.osc = (int)i; int32_t cur = prog_[i].dst; ++i;
        if (i < n && (prog_[i].op == MXB_OP_ENV_ADSR || prog_[i].op == MXB_OP_ENV_AR)) {
            const mxb_stage& g = prog_[i];
            if (g.src[0] != cur || gateInput_ < 0 || g.src[1] != MXB_INPUT(gateInput_) || !args_const(g, 2)) return false;
            c.env = (int)i; cur = g.dst; ++i;
        }
        if (i < n && (prog_[i].op == MXB_OP_FILTER || prog_[i].op == MXB_OP_SVF || prog_[i].op == MXB_OP_BIQUAD)) {
            const mxb_stage& g = prog_[i];
            if (g.src[0] != cur || !args_const(g, 1)) return false;
            if (g.op == MXB_OP_FILTER && g.kind != MXB_FILT_LORES && g.kind != MXB_FILT_HIRES) return false;
            if (g.op == MXB_OP_SVF) for (int k = 3; k < 7; ++k) if ((g.src[k] >> 8) != 2) return false;      /* mix weights: constants */
            c.filt = (int)i; cur = g.dst; ++i;
        }
        if (i < n && prog_[i].op == MXB_OP_DELAY) {
            const mxb_stage& g = prog_[i];
            if (g.src[0] != cur || !args_const(g, 1)) return false;
            c.dly = (int)i; cur = g.dst; ++i;
        }
        for (; i < n; ++i) {
            const mxb_stage& g = prog_[i];
            if (g.op == MXB_OP_MIX_STEREO && c.mix < 0 && g.src[0] == cur && blockConstant(g.src[1])) c.mix = (int)i;
            else if (g.op == MXB_OP_OUT && c.out < 0 && g.src[0] == cur) c.out = (int)i;
            else return false;
        }
        return nInputs_ == (c.env >= 0 ? 1 : 0);
    }

    void build(int nFrames) {
        using maxib200_detail::check;
        const int maxFrames = nFrames > (int)maxiSettings::bufferSize ? nFrames : (int)maxiSettings::bufferSize;
        Chain c;
        if (matchChain(c)) {
            mxb_bank_desc d;
            std::memset(&d, 0, sizeof(d));
            d.voices = V_; d.max_frames = maxFrames; d.osc_kind = prog_[(size_t)c.osc].kind;
            if (c.env >= 0) d.env_kind = prog_[(size_t)c.env].op == MXB_OP_ENV_ADSR ? MXB_ENV_ADSR : MXB_ENV_AR;
            if (c.filt >= 0) {
                const mxb_stage& g = prog_[(size_t)c.filt];
                d.filt_kind = g.op == MXB_OP_SVF ? MXB_FILT_SVF : g.op == MXB_OP_BIQUAD ? MXB_FILT_BIQUAD : g.kind;
                if (g.op == MXB_OP_BIQUAD) d.biquad_type = g.kind;
                if (g.op == MXB_OP_SVF) for (int k = 0; k < 4; ++k) d.svf_mix[k] = consts_[(size_t)(g.src[3 + k] & 0xff)];
            }
            if (c.dly >= 0) { d.delay_taps = delayCapacity_ > 0 ? delayCapacity_ : taps_; d.delay_mode = prog_[(size_t)c.dly].kind; }
            check(mxb_bank_create(ctx_, &d, &bank_), "mxb_bank_create");
            chain_ = c;
        } else {
            if (haveTables_) check(mxb_ctx_set_tables(ctx_, sine_.data(), trans_.data(), sineBefore_), "mxb_ctx_set_tables");
            mxb_patch_desc d;
            std::memset(&d, 0, sizeof(d));
            d.voices = V_; d.n_stages = (int32_t)prog_.size(); d.n_params = nParams_; d.n_consts = (int32_t)consts_.size(); d.n_inputs = nInputs_;
            d.max_frames = maxFrames; d.delay_taps = delayCapacity_ > 0 ? delayCapacity_ : taps_;
            d.stages = prog_.data(); d.consts = consts_.data(); d.input_types = inputType_.data();
            std::vector<mxb_envgen_shape> shapes;
            for (const EgShape& s : egShapes_) shapes.push_back({(int32_t)s.times.size(), s.loop, s.retrigger, s.levels.data(), s.times.data(), s.curves.data()});
            check(mxb_patch_create2(ctx_, &d, (int32_t)shapes.size(), shapes.data(), &patch_), "mxb_patch_create2");
        }
        built_ = prog_; builtConsts_ = consts_; builtShapes_ = egShapes_; builtTypes_.assign(inputType_.begin(), inputType_.begin() + nInputs_);
        for (size_t j = 0; j < paramDirty_.size(); ++j) paramDirty_[j] = true;
    }

    void setBank(int id, int32_t s) {
        if (s == MXB_NONE) return;
        const bool isParam = (s >> 8) == 1;
        if (isParam && !paramDirty_[(size_t)(s & 0xff)] && bankSet_[id]) return;
        if (!isParam && bankSet_[id]) return;                         /* constants never change (sameProgram) */
        const std::vector<double> v = values(s);
        maxib200_detail::check(mxb_bank_set_param(bank_, id, v.data(), MXB_MEM_HOST), "mxb_bank_set_param");
        bankSet_[id] = true;
    }
    void runBank(int nFrames, double* out, double* mix) {
        const Chain& c = chain_;
        const mxb_stage& o = prog_[(size_t)c.osc];
        if (o.kind == MXB_OSC_PULSE) setBank(MXB_P_DUTY, o.src[1]);
        if (o.kind == MXB_OSC_PHASORBETWEEN) { setBank(MXB_P_PHASOR_START, o.src[1]); setBank(MXB_P_PHASOR_END, o.src[2]); }
        setBank(MXB_P_FREQ, o.src[0]);
        for (const auto& ph : pendingPhase_) maxib200_detail::check(mxb_bank_set_param(bank_, MXB_P_PHASE, ph.second.data(), MXB_MEM_HOST), "mxb_bank_set_param");
        if (c.env >= 0) {
            const mxb_stage& g = prog_[(size_t)c.env];
            if (g.op == MXB_OP_ENV_ADSR) { setBank(MXB_P_ENV_ATTACK, g.src[2]); setBank(MXB_P_ENV_DECAY, g.src[3]); setBank(MXB_P_ENV_SUSTAIN, g.src[4]);
                                           setBank(MXB_P_ENV_RELEASE, g.src[5]); setBank(MXB_P_ENV_HOLDTIME, g.src[6]); }
            else { setBank(MXB_P_ENV_ATTACK, g.src[2]); setBank(MXB_P_ENV_RELEASE, g.src[3]); setBank(MXB_P_ENV_HOLDTIME, g.src[4]); }
        }
        if (c.filt >= 0) {
            const mxb_stage& g = prog_[(size_t)c.filt];
            if (g.op == MXB_OP_BIQUAD) setBank(MXB_P_GAIN, g.src[3]);
            setBank(MXB_P_CUTOFF, g.src[1]); setBank(MXB_P_RESONANCE, g.src[2]);
        }
        if (c.dly >= 0) {
            const mxb_stage& g = prog_[(size_t)c.dly];
            setBank(MXB_P_DELAY_SIZE, g.src[1]); setBank(MXB_P_DELAY_FEEDBACK, g.src[2]);
            if (g.kind == MXB_DELAY_FROM_POSITION) setBank(MXB_P_DELAY_POSITION, g.src[3]);
        }
        if (c.mix >= 0) setBank(MXB_P_PAN, prog_[(size_t)c.mix].src[1]);
        for (size_t j = 0; j < paramDirty_.size(); ++j) paramDirty_[j] = false;
        const int32_t* on = gate_.on ? gate_.on->data() : nullptr;
        const int32_t* off = gate_.off ? gate_.off->data() : nullptr;
        maxib200_detail::check(mxb_bank_process(bank_, nFrames, on, off, c.out >= 0 ? out : nullptr, MXB_F64, c.mix >= 0 ? mix : nullptr, MXB_MEM_HOST, nullptr),
                               "mxb_bank_process");
    }
    void runPatch(int nFrames, double* out, double* mix) {
        using maxib200_detail::check;
        for (int j = 0; j < nParams_; ++j) {
            if (!paramDirty_[(size_t)j]) continue;
            check(mxb_patch_set_param(patch_, j, paramVals_[(size_t)j].data(), MXB_MEM_HOST), "mxb_patch_set_param");
            paramDirty_[(size_t)j] = false;
        }
        for (const auto& ph : pendingPhase_) check(mxb_patch_set_state(patch_, ph.first, 0, ph.second.data(), MXB_MEM_HOST), "mxb_patch_set_state");
        if (gateInput_ >= 0) {        /* the interval gate as a per-sample trigger stream */
            gateStream_.assign((size_t)nFrames * (size_t)V_, 0.0);
            if (gate_.on && gate_.off)
                for (int v = 0; v < V_; ++v)
                    for (int t = (*gate_.on)[(size_t)v] < 0 ? 0 : (*gate_.on)[(size_t)v]; t < (*gate_.off)[(size_t)v] && t < nFrames; ++t) gateStream_[(size_t)t * (size_t)V_ + (size_t)v] = 1.0;
            inputPtr_[(size_t)gateInput_] = gateStream_.data();
        }
        for (int k = 0; k < nInputs_; ++k) if (inputEv_[(size_t)k]) inputPtr_[(size_t)k] = inputEv_[(size_t)k]->pack();
        check(mxb_patch_process(patch_, nFrames, nInputs_ ? (const void* const*)inputPtr_.data() : nullptr, outSrc_ != MXB_NONE ? out : nullptr, wantMix_ ? mix : nullptr,
                                MXB_MEM_HOST, nullptr), "mxb_patch_process");
    }

    friend class maxiOsc; friend class maxiEnvGen;
    int V_, device_, taps_ = 0;
    mxb_ctx* ctx_ = nullptr;
    mxb_bank* bank_ = nullptr;
    mxb_patch* patch_ = nullptr;
    std::vector<mxb_stage> prog_, built_;
    std::vector<double> consts_, builtConsts_;
    std::vector<std::vector<double>> paramVals_;
    std::vector<bool> paramDirty_;
    std::vector<const void*> inputPtr_;           /* per input stream: its data (an mxb_events for an events stream), type and maxiEvents */
    std::vector<int32_t> inputType_, builtTypes_;
    std::vector<maxiEvents*> inputEv_;
    std::vector<double> gateStream_;
    std::vector<std::pair<int, std::vector<double>>> pendingPhase_;      /* maxiOsc::phaseReset: (stage, per-voice phase), applied before the block */
    std::vector<const void*> egObjs_;                                     /* the maxiEnvGen objects that played in this block, by shape index */
    std::vector<EgShape> egShapes_, builtShapes_;
    std::vector<double> sine_, trans_; double sineBefore_ = 0.0; bool haveTables_ = false;
    int nParams_ = 0, nInputs_ = 0, nextReg_ = 0, gateInput_ = -1;
    int32_t outSrc_ = MXB_NONE, lastSrc_ = MXB_NONE;
    bool wantMix_ = false;
    bool bankSet_[MXB_P_COUNT] = {};
    maxiGate gate_;
    Chain chain_;
};

inline maxiEvents::maxiEvents(maxiVoices& v) : v_(&v), V_(v.size()) {}

/* the arithmetic a play() does between the calls: recorded like everything else */
namespace maxib200_detail {
inline maxiSignal bin(int32_t op, maxiVoices* v, int32_t a, int32_t b) { return v->emit(op, 0, {a, b}); }
}
inline maxiSignal operator+(maxiSignal a, maxiSignal b) { a.voices->check(b, "operator+"); return maxib200_detail::bin(MXB_OP_ADD, a.voices, a.src, b.src); }
inline maxiSignal operator-(maxiSignal a, maxiSignal b) { a.voices->check(b, "operator-"); return maxib200_detail::bin(MXB_OP_SUB, a.voices, a.src, b.src); }
inline maxiSignal operator*(maxiSignal a, maxiSignal b) { a.voices->check(b, "operator*"); return maxib200_detail::bin(MXB_OP_MUL, a.voices, a.src, b.src); }
inline maxiSignal operator/(maxiSignal a, maxiSignal b) { a.voices->check(b, "operator/"); return maxib200_detail::bin(MXB_OP_DIV, a.voices, a.src, b.src); }
inline maxiSignal operator+(maxiSignal a, const maxiParam& b) { return maxib200_detail::bin(MXB_OP_ADD, a.voices, a.src, a.voices->operand(b)); }
inline maxiSignal operator-(maxiSignal a, const maxiParam& b) { return maxib200_detail::bin(MXB_OP_SUB, a.voices, a.src, a.voices->operand(b)); }
inline maxiSignal operator*(maxiSignal a, const maxiParam& b) { return maxib200_detail::bin(MXB_OP_MUL, a.voices, a.src, a.voices->operand(b)); }
inline maxiSignal operator/(maxiSignal a, const maxiParam& b) { return maxib200_detail::bin(MXB_OP_DIV, a.voices, a.src, a.voices->operand(b)); }
inline maxiSignal operator+(const maxiParam& a, maxiSignal b) { return maxib200_detail::bin(MXB_OP_ADD, b.voices, b.voices->operand(a), b.src); }
inline maxiSignal operator-(const maxiParam& a, maxiSignal b) { return maxib200_detail::bin(MXB_OP_SUB, b.voices, b.voices->operand(a), b.src); }
inline maxiSignal operator*(const maxiParam& a, maxiSignal b) { return maxib200_detail::bin(MXB_OP_MUL, b.voices, b.voices->operand(a), b.src); }
inline maxiSignal operator/(const maxiParam& a, maxiSignal b) { return maxib200_detail::bin(MXB_OP_DIV, b.voices, b.voices->operand(a), b.src); }

/* An argument of a stage: a signal computed earlier in play(), or a parameter. */
class maxiArg {
public:
    maxiArg(maxiSignal s) : sig_(s), isSig_(true) {}
    maxiArg(double v) : par_(v) {}
    maxiArg(int v) : par_((double)v) {}
    maxiArg(const std::vector<double>& v) : par_(v) {}
    maxiArg(const maxiParam& p) : par_(p) {}
    maxiArg(const maxiStream& s) : stream_(s.values), isStream_(true) {}
    maxiArg(const maxiEvents& e) : ev_(&e) {}
    int32_t op(maxiVoices* v) const {
        if (isSig_) { v->check(sig_, "argument"); return sig_.src; }
        if (isStream_) return v->operand(maxiStream(stream_));
        if (ev_) return v->operand(*ev_);
        return v->operand(par_);
    }
private:
    maxiSignal sig_; maxiParam par_; bool isSig_ = false;
    const double* stream_ = nullptr; bool isStream_ = false;
    const maxiEvents* ev_ = nullptr;
};

/* maxiOsc, src/maximilian.h:169-215 / src/maximilian.cpp:209-373 */
class maxiOsc {
public:
    explicit maxiOsc(maxiVoices& v) : v_(&v) {}
    maxiSignal sinewave(const maxiArg& frequency) { return osc(MXB_OSC_SINEWAVE, frequency); }
    maxiSignal coswave(const maxiArg& frequency) { return osc(MXB_OSC_COSWAVE, frequency); }
    maxiSignal phasor(const maxiArg& frequency) { return osc(MXB_OSC_PHASOR, frequency); }
    maxiSignal saw(const maxiArg& frequency) { return osc(MXB_OSC_SAW, frequency); }
    maxiSignal square(const maxiArg& frequency) { return osc(MXB_OSC_SQUARE, frequency); }
    maxiSignal triangle(const maxiArg& frequency) { return osc(MXB_OSC_TRIANGLE, frequency); }
    maxiSignal impulse(const maxiArg& frequency) { return osc(MXB_OSC_IMPULSE, frequency); }
    maxiSignal sinebuf(const maxiArg& frequency) { return osc(MXB_OSC_SINEBUF, frequency); }
    maxiSignal sinebuf4(const maxiArg& frequency) { return osc(MXB_OSC_SINEBUF4, frequency); }
    maxiSignal sawn(const maxiArg& frequency) { return osc(MXB_OSC_SAWN, frequency); }
    maxiSignal pulse(const maxiArg& frequency, const maxiArg& duty) { return emitOsc(MXB_OSC_PULSE, {frequency.op(v_), duty.op(v_)}); }
    maxiSignal phasorBetween(const maxiArg& frequency, const maxiArg& startphase, const maxiArg& endphase) {
        return emitOsc(MXB_OSC_PHASORBETWEEN, {frequency.op(v_), startphase.op(v_), endphase.op(v_)});
    }
    /* maxiOsc::phaseReset (src/maximilian.cpp:222-226): takes effect before the next block this oscillator plays in */
    void phaseReset(const maxiParam& phaseIn) { pending_ = phaseIn.isScalar() ? std::vector<double>((size_t)v_->size(), phaseIn.scalar()) : phaseIn.vec(); }
private:
    maxiSignal osc(int kind, const maxiArg& f) { return emitOsc(kind, {f.op(v_)}); }
    maxiSignal emitOsc(int kind, std::initializer_list<int32_t> srcs) {
        if (!pending_.empty()) { v_->pendingPhase_.emplace_back((int)v_->prog_.size(), pending_); pending_.clear(); }
        return v_->emit(MXB_OP_OSC, kind, srcs, true, 1);
    }
    maxiVoices* v_;
    std::vector<double> pending_;
};

/* maxiFilter, src/maximilian.cpp:442-500 */
class maxiFilter {
public:
    explicit maxiFilter(maxiVoices& v) : v_(&v) {}
    maxiSignal lores(maxiSignal input, const maxiArg& cutoff1, const maxiArg& resonance) { return f(MXB_FILT_LORES, input, cutoff1, resonance); }
    maxiSignal hires(maxiSignal input, const maxiArg& cutoff1, const maxiArg& resonance) { return f(MXB_FILT_HIRES, input, cutoff1, resonance); }
    maxiSignal bandpass(maxiSignal input, const maxiArg& cutoff1, const maxiArg& resonance) { return f(MXB_FILT_BANDPASS, input, cutoff1, resonance); }
    maxiSignal lopass(maxiSignal input, const maxiArg& cutoff) { v_->check(input, "maxiFilter::lopass"); return v_->emit(MXB_OP_FILTER, MXB_FILT_LOPASS, {input.src, cutoff.op(v_)}, true, 3); }
    maxiSignal hipass(maxiSignal input, const maxiArg& cutoff) { v_->check(input, "maxiFilter::hipass"); return v_->emit(MXB_OP_FILTER, MXB_FILT_HIPASS, {input.src, cutoff.op(v_)}, true, 3); }
private:
    maxiSignal f(int kind, maxiSignal in, const maxiArg& c, const maxiArg& r) {
        v_->check(in, "maxiFilter");
        return v_->emit(MXB_OP_FILTER, kind, {in.src, c.op(v_), r.op(v_)}, true, 3);
    }
    maxiVoices* v_;
};

/* maxiSVF, src/maximilian.h:1281-1338 */
class maxiSVF {
public:
    explicit maxiSVF(maxiVoices& v) : v_(&v) {}
    void setCutoff(const maxiArg& cutoff) { cutoff_ = cutoff; }
    void setResonance(const maxiArg& q) { res_ = q; }
    maxiSignal play(maxiSignal w, double lpmix, double bpmix, double hpmix, double notchmix) {
        v_->check(w, "maxiSVF::play");
        return v_->emit(MXB_OP_SVF, 0, {w.src, cutoff_.op(v_), res_.op(v_), v_->constOp(lpmix), v_->constOp(bpmix), v_->constOp(hpmix), v_->constOp(notchmix)}, true, 3);
    }
private:
    maxiVoices* v_;
    maxiArg cutoff_{1000.0}, res_{1.0};        /* maxiSVF ctor: setParams(1000, 1), src/maximilian.h:1284 */
};

/* maxiBiquad, src/maximilian.h:1343-1486. The reference's constructor designs nothing: until set() runs, every coefficient is 0
 * (:1482) and play() returns 0 while its state follows the input. No stage computes that, so play() before set() throws
 * maxiError(MXB_ERR_UNSUPPORTED) instead of inventing a design. */
class maxiBiquad {
public:
    enum filterTypes { LOWPASS, HIGHPASS, BANDPASS, NOTCH, PEAK, LOWSHELF, HIGHSHELF };
    explicit maxiBiquad(maxiVoices& v) : v_(&v) {}
    void set(filterTypes filtType, const maxiArg& cutoff, const maxiArg& Q, const maxiArg& peakGain) {
        type_ = (int)filtType; cutoff_ = cutoff; q_ = Q; gain_ = peakGain; set_ = true;
    }
    maxiSignal play(maxiSignal input) {
        v_->check(input, "maxiBiquad::play");
        if (!set_) throw maxiError(MXB_ERR_UNSUPPORTED, "maxiBiquad::play: set() was never called (the reference's coefficients are all 0)");
        return v_->emit(MXB_OP_BIQUAD, type_, {input.src, cutoff_.op(v_), q_.op(v_), gain_.op(v_)}, true, 3);
    }
private:
    maxiVoices* v_;
    int type_ = 0;
    bool set_ = false;
    maxiArg cutoff_{0.0}, q_{0.0}, gain_{0.0};
};

/* maxiEnv (ADSR / AR), src/maximilian.h:888-932 / src/maximilian.cpp:1319-1494. The trigger is an argument here (the reference's
 * public member `trigger`, written by the patch on any sample): a maxiGate interval or a maxiStream of per-sample values. */
class maxiEnv {
public:
    explicit maxiEnv(maxiVoices& v) : v_(&v) {}
    void setAttack(const maxiParam& attackMS) { coeff(0, 0, attackMS); }
    void setAttackMS(const maxiParam& attackMS) { coeff(0, 1, attackMS); }
    void setDecay(const maxiParam& decayMS) { coeff(1, 2, decayMS); }
    void setRelease(const maxiParam& releaseMS) { coeff(3, 2, releaseMS); }
    void setSustain(const maxiParam& sustainL) { set(2, sustainL); }
    void setHoldtime(const maxiParam& holdtime) { set(4, holdtime); }          /* the public member `holdtime` (default 1) */
    template <class Trig> maxiSignal adsr(const maxiArg& input, const Trig& trigger) {
        return v_->emit(MXB_OP_ENV_ADSR, 0, {input.op(v_), v_->operand(trigger), arg(0), arg(1), arg(2), arg(3), arg(4)}, true, 2);
    }
    /* the overload that takes the raw coefficients as arguments (src/maximilian.cpp:1362-1413): the same state machine */
    template <class Trig> maxiSignal adsr(const maxiArg& input, const maxiParam& attack, const maxiParam& decay, const maxiParam& sustain, const maxiParam& release,
                                         const maxiParam& holdtime, const Trig& trigger) {
        set(0, attack); set(1, decay); set(2, sustain); set(3, release); set(4, holdtime);
        return adsr(input, trigger);
    }
    /* maxiEnv::ar(input, attack, release, holdtime, trigger): attack / release are the raw per-sample coefficients */
    template <class Trig> maxiSignal ar(const maxiArg& input, const maxiParam& attack, const maxiParam& release, const maxiParam& holdtime, const Trig& trigger) {
        return v_->emit(MXB_OP_ENV_AR, 0, {input.op(v_), v_->operand(trigger), v_->operand(attack), v_->operand(release), v_->operand(holdtime)}, true, 2);
    }
private:
    void set(int k, const maxiParam& p) { scalar_[k] = p.isScalar(); if (p.isScalar()) val_[k] = p.scalar(); else vec_[k] = p.vec(); }
    int32_t arg(int k) { return scalar_[k] ? v_->constOp(val_[k]) : v_->operand(maxiParam(vec_[k])); }
    void coeff(int k, int kind, const maxiParam& ms) {
        std::vector<double> in = ms.isScalar() ? std::vector<double>(1, ms.scalar()) : ms.vec();
        std::vector<double> out(in.size());
        maxib200_detail::check(mxb_env_coeffs(kind, in.data(), (int64_t)in.size(), (int32_t)maxiSettings::sampleRate, out.data()), "mxb_env_coeffs");
        if (ms.isScalar()) set(k, maxiParam(out[0])); else set(k, maxiParam(out));
    }
    maxiVoices* v_;
    bool scalar_[5] = {true, true, true, true, true};
    double val_[5] = {0, 0, 0, 0, 1.0};          /* maxiEnv: zero-filled but holdtime = 1, src/maximilian.h:913 */
    std::vector<double> vec_[5];
};

/* maxiEnvGen, src/maximilian.h:2268-2547: each object owns its envelope shape (levels, times, curves, loop, retrigger), played by all voices,
 * each voice with its own state. An object whose setup() was never called plays 0, as in the reference. The shape is part of the patch: a
 * shape changed after the first block is a different patch (maxiVoices::render throws). */
class maxiEnvGen {
public:
    static constexpr double HOLD = MXB_ENVGEN_HOLD;
    explicit maxiEnvGen(maxiVoices& v) : v_(&v) {}
    bool setup(const std::vector<double>& levels, const std::vector<double>& times, const std::vector<double>& curves, bool looping, bool allowRetrigger = false) {
        if (levels.size() != times.size() + 1 || levels.size() != curves.size() + 1) return false;
        size_t n = times.size();
        bool hold = false;
        for (size_t i = 0; i < times.size() && n == times.size(); ++i) {
            if (times[i] == HOLD && hold) n = i;
            hold = hold || times[i] == HOLD;
        }
        /* the reference stops at a second HOLD segment (returns false), keeping the segments before it and the old loop / retrigger */
        shape_.levels.assign(levels.begin(), levels.begin() + (long)n + 1);
        shape_.times.assign(times.begin(), times.begin() + (long)n);
        shape_.curves.assign(curves.begin(), curves.begin() + (long)n);
        if (n < times.size()) return false;
        shape_.loop = looping; shape_.retrigger = allowRetrigger;
        return true;
    }
    void setLoop(const bool val) { shape_.loop = val; }
    bool getLoop() { return shape_.loop != 0; }
    void setRetrigger(const bool val) { shape_.retrigger = val; }
    bool getRetrigger() { return shape_.retrigger != 0; }
    void setupAR(double attack, double release) { setup({0, 1, 0}, {attack, release}, {1, 1}, false, false); }
    void setupASR(double attack, double release) { setup({0, 1, 1, 0}, {attack, HOLD, release}, {1, 1, 1}, false, false); }
    void setupADSR(double attack, double decay, double sustain, double release) { setup({0, 1, sustain, sustain, 0}, {attack, decay, HOLD, release}, {1, 1, 1, 1}, false, false); }
    template <class Trig> maxiSignal play(const Trig& trigger) { const int32_t t = trig(trigger); return v_->emit(MXB_OP_ENVGEN, v_->egShape(this, shape_), {t}); }
private:
    int32_t trig(const maxiSignal& s) { v_->check(s, "maxiEnvGen::play"); return s.src; }
    int32_t trig(const maxiStream& s) { return v_->operand(s); }
    int32_t trig(const maxiEvents& e) { return v_->operand(e); }
    int32_t trig(const maxiParam& p) { return v_->operand(p); }
    maxiVoices* v_;
    maxiVoices::EgShape shape_;
};

/* maxiDelayline, src/maximilian.h:266-284 / src/maximilian.cpp:415-439 */
class maxiDelayline {
public:
    /* capacity: ring slots per voice (the reference allocates 705600 for every object) */
    maxiDelayline(maxiVoices& v, int capacity) : v_(&v), capacity_(capacity) {}
    maxiSignal dl(maxiSignal input, const maxiArg& size, const maxiArg& feedback) {
        v_->check(input, "maxiDelayline::dl"); v_->delayCapacity_ = capacity_;
        return v_->emit(MXB_OP_DELAY, MXB_DELAY_DL, {input.src, size.op(v_), feedback.op(v_)}, true, 4);
    }
    maxiSignal dlFromPosition(maxiSignal input, const maxiArg& size, const maxiArg& feedback, const maxiArg& position) {
        v_->check(input, "maxiDelayline::dlFromPosition"); v_->delayCapacity_ = capacity_;
        return v_->emit(MXB_OP_DELAY, MXB_DELAY_FROM_POSITION, {input.src, size.op(v_), feedback.op(v_), position.op(v_)}, true, 4);
    }
private:
    maxiVoices* v_;
    int capacity_;
};

/* maxiFlanger, src/maximilian.h:1144-1180 */
class maxiFlanger {
public:
    maxiFlanger(maxiVoices& v, int capacity) : v_(&v), capacity_(capacity) {}
    maxiSignal flange(maxiSignal input, const maxiArg& delay, const maxiArg& feedback, const maxiArg& speed, const maxiArg& depth) {
        v_->check(input, "maxiFlanger::flange"); v_->delayCapacity_ = capacity_;
        return v_->emit(MXB_OP_FLANGER, 0, {input.src, delay.op(v_), feedback.op(v_), speed.op(v_), depth.op(v_)});
    }
private:
    maxiVoices* v_;
    int capacity_;
};

/* maxiChorus, src/maximilian.h:1180-1212. The reference draws its modulator from libc rand() inside the call (lfo.noise()); here the caller
 * owns the random stream and hands over what noise() would have returned for every sample of the block -- maxiStream of
 * [frame][voice] values in [-1, 1], e.g. `float r = rand() / (float)RAND_MAX; x = r * 2 - 1;` in frame-major order to replay the
 * reference exactly. Everything after the draw (the lores-filtered modulator, both swept delay lines, the normalisation) is the stage. */
class maxiChorus {
public:
    maxiChorus(maxiVoices& v, int capacity) : v_(&v), capacity_(capacity) {}
    template <class Noise>      /* maxiStream or maxiEvents */
    maxiSignal chorus(maxiSignal input, const maxiArg& delay, const maxiArg& feedback, const maxiArg& speed, const maxiArg& depth, const Noise& noise) {
        v_->check(input, "maxiChorus::chorus"); v_->delayCapacity_ = capacity_;
        return v_->emit(MXB_OP_CHORUS, 0, {input.src, delay.op(v_), feedback.op(v_), speed.op(v_), depth.op(v_), v_->operand(noise)});
    }
private:
    maxiVoices* v_;
    int capacity_;
};

/* maxiDCBlocker, src/maximilian.h:1255-1267 */
class maxiDCBlocker {
public:
    explicit maxiDCBlocker(maxiVoices& v) : v_(&v) {}
    maxiSignal play(maxiSignal input, const maxiArg& R) { v_->check(input, "maxiDCBlocker::play"); return v_->emit(MXB_OP_DCBLOCK, 0, {input.src, R.op(v_)}); }
private:
    maxiVoices* v_;
};

/* maxiNonlinearity, src/maximilian.h:1046-1137 */
class maxiNonlinearity {
public:
    explicit maxiNonlinearity(maxiVoices& v) : v_(&v) {}
    maxiSignal atanDist(maxiSignal in, const maxiArg& shape) { return nl(MXB_NL_ATANDIST, in, shape.op(v_), MXB_NONE); }
    maxiSignal fastAtanDist(maxiSignal in, const maxiArg& shape) { return nl(MXB_NL_FASTATANDIST, in, shape.op(v_), MXB_NONE); }
    maxiSignal softclip(maxiSignal x) { return nl(MXB_NL_SOFTCLIP, x, MXB_NONE, MXB_NONE); }
    maxiSignal hardclip(maxiSignal x) { return nl(MXB_NL_HARDCLIP, x, MXB_NONE, MXB_NONE); }
    maxiSignal asymclip(maxiSignal x, const maxiArg& a, const maxiArg& b) { return nl(MXB_NL_ASYMCLIP, x, a.op(v_), b.op(v_)); }
    maxiSignal fastatan(maxiSignal x) { return nl(MXB_NL_FASTATAN, x, MXB_NONE, MXB_NONE); }
private:
    maxiSignal nl(int kind, maxiSignal x, int32_t p1, int32_t p2) { v_->check(x, "maxiNonlinearity"); return v_->emit(MXB_OP_NONLIN, kind, {x.src, p1, p2}); }
    maxiVoices* v_;
};
using maxiDistortion = maxiNonlinearity;       /* src/maximilian.h:1139 */

/* maxiMix::stereo, src/maximilian.h:400 / src/maximilian.cpp:503-509; the per-voice results are summed into the bus */
class maxiMix {
public:
    explicit maxiMix(maxiVoices& v) : v_(&v) {}
    void stereo(maxiSignal input, maxiBus two, const maxiArg& x) {
        if (two.voices != v_) throw maxiError(MXB_ERR_UNSUPPORTED, "maxiMix::stereo: signal and bus must belong to the same maxiVoices");
        v_->check(input, "maxiMix::stereo");
        v_->emit(MXB_OP_MIX_STEREO, 0, {input.src, x.op(v_)}, false);
    }
private:
    maxiVoices* v_;
};

/* ---- block-dispatch shim: stands in for routing() of cpp/commandline/player.cpp:25-44 (RtAudio callback signature,
 * cpp/commandline/RtAudio.h:205-209). The user supplies  void play(maxiVoices&)  -- the block-rate twin of the
 * reference's  void play(double*)  -- and passes the maxiVoices as userData; the interleaved RTAUDIO_FLOAT64
 * stereo buffer is exactly the patch's mix bus. ---- */
void play(maxiVoices& voices);
inline int maxiRouting(void* outputBuffer, void* /*inputBuffer*/, unsigned int nBufferFrames, double /*streamTime*/,
                       unsigned int /*status*/, void* userData) {
    maxiVoices* v = static_cast<maxiVoices*>(userData);
    play(*v);
    v->render((int)nBufferFrames, nullptr, static_cast<double*>(outputBuffer));
    return 0;
}

/* ---- spectral classes: C channels at once ---- */

/* maxiMFCC, src/libs/maxiMFCC.h:40-211 */
class maxiMFCC {
public:
    maxiMFCC() {}
    ~maxiMFCC() { if (h_) mxb_mfcc_destroy(h_); if (ctx_) mxb_ctx_destroy(ctx_); }
    maxiMFCC(const maxiMFCC&) = delete;
    void setup(unsigned int numBins, unsigned int numFilters, unsigned int numCoeffs, double minFreq, double maxFreq, int device = 0) {
        using maxib200_detail::check;
        check(mxb_ctx_create(device, (int32_t)maxiSettings::sampleRate, &ctx_), "mxb_ctx_create");
        check(mxb_mfcc_create(ctx_, (int32_t)numBins, (int32_t)numFilters, (int32_t)numCoeffs, minFreq, maxFreq, &h_), "mxb_mfcc_create");
        bins_ = (int)numBins; coeffs_ = (int)numCoeffs;
    }
    /* powerSpectrum: frames x numBins magnitudes (host); returns frames x numCoeffs */
    std::vector<double>& mfcc(const std::vector<float>& powerSpectrum) {
        const int64_t n = (int64_t)(powerSpectrum.size() / (size_t)bins_);
        out_.resize((size_t)n * (size_t)coeffs_);
        maxib200_detail::check(mxb_mfcc_process(h_, powerSpectrum.data(), n, out_.data(), nullptr, MXB_MEM_HOST, nullptr), "mxb_mfcc_process");
        return out_;
    }
    mxb_mfcc* handle() { return h_; }
private:
    mxb_ctx* ctx_ = nullptr; mxb_mfcc* h_ = nullptr; int bins_ = 0, coeffs_ = 0;
    std::vector<double> out_;
};

class maxiFFT;

/* maxiFFTOctaveAnalyzer, src/libs/maxiFFT.h:162-205, maxiFFT.cpp:201-300, used in either of two ways:
 *  - attached to a maxiFFT (fft.attach(oct), before or after setup()): the transform's process() runs calculate() for every frame it
 *    fires, on the device (fused into the transform at fft size 1024; at other sizes mxb_octave_process on the magnitudes it just wrote).
 *    `averages` / `peaks` point at the LAST fired frame of channel 0 (what a reference patch reads after calculate()), averagesOf(c, f) /
 *    peaksOf(c, f) at any frame of the last call. calculate(fftData) accepts the attached transform's own magnitudes (the values are
 *    already there) and rejects any other pointer: process() has already run calculate() for that frame. nBandsInTheFFT must be the
 *    transform's getNumBins(): process() refuses any other count with MXB_ERR_INVALID, at every fft size (the reference would read
 *    past the magnitudes, or the wrong bins of every frame but the first).
 *  - not attached: calculate(fftData) analyses the nBandsInTheFFT magnitudes it is handed, one frame per call (a host shim over
 *    mxb_octave_process on the analyser's own context, like the per-sample maxiFFT::process), and points `averages` / `peaks` at the result.
 * The public members keep the reference's names: peakHoldTime, peakDecayRate, linearEQIntercept and linearEQSlope are read at every
 * process() / calculate(). nAverages is known after setup() (for an attached analyser, once its transform is set up too). The analyser
 * owns device handles, so unlike the reference's class it cannot be copied. */
class maxiFFTOctaveAnalyzer {
public:
    float samplingRate = 0.f;
    int nSpectrum = 0, nAverages = 0, nAveragesPerOctave = 0;
    float* averages = nullptr;
    float* peaks = nullptr;
    int peakHoldTime = 0;                                   /* setup()'s values, src/libs/maxiFFT.cpp:257-261 */
    float peakDecayRate = 0.9f, linearEQIntercept = 1.0f, linearEQSlope = 0.0f;
    maxiFFTOctaveAnalyzer() {}
    ~maxiFFTOctaveAnalyzer() { if (h_) mxb_octave_destroy(h_); if (ctx_) mxb_ctx_destroy(ctx_); }
    maxiFFTOctaveAnalyzer(const maxiFFTOctaveAnalyzer&) = delete;
    /* device: where an analyser that is not attached computes */
    void setup(float samplingRate_, int nBandsInTheFFT, int nAveragesPerOctave_, int device = 0) {
        samplingRate = samplingRate_; nSpectrum = nBandsInTheFFT; nAveragesPerOctave = nAveragesPerOctave_ == 0 ? 1 : nAveragesPerOctave_;
        peakHoldTime = 0; peakDecayRate = 0.9f; linearEQIntercept = 1.0f; linearEQSlope = 0.0f;
        device_ = device;
        isSetup_ = true;
        create();
    }
    inline void calculate(const float* fftData);
    const float* averagesOf(int channel, int frame) const { return avg_.data() + ((size_t)channel * (size_t)maxf_ + (size_t)frame) * (size_t)nAverages; }
    const float* peaksOf(int channel, int frame) const { return pk_.data() + ((size_t)channel * (size_t)maxf_ + (size_t)frame) * (size_t)nAverages; }
private:
    friend class maxiFFT;
    inline void create();
    maxiFFT* fft_ = nullptr;
    mxb_ctx* ctx_ = nullptr;                                /* not attached: the analyser's own */
    mxb_octave* h_ = nullptr;
    bool isSetup_ = false;
    int device_ = 0, maxf_ = 0;
    std::vector<float> avg_, pk_;
};

/* maxiBarkScaleAnalyser / maxiBark, src/libs/maxiBark.h:36-128, likewise in either of two ways:
 *  - attached to a maxiFFT (fft.attach(bark)); setup(sR, bS) must name the transform's own sample rate and size. specificLoudness /
 *    relativeLoudness / totalLoudness return the values of the LAST fired frame of channel 0 and accept the attached transform's
 *    magnitudes only (any other pointer is rejected); ...Of(c, f) reach the rest.
 *  - not attached: each of the three computes on the bS / 2 values it is handed (one frame per call, mxb_bark_process on the analyser's
 *    own context) and returns the result.
 * The analyser's own context and mxb_bark handle are created on first use, i.e. never for an analyser attached to a 1024-point
 * transform (its kernel computes the loudness itself); the reference's limits (bS in 2 .. 4096, bin * sR within unsigned int) are
 * checked then. The analyser owns device handles, so unlike the reference's class it cannot be copied. */
template <class T>
class maxiBarkScaleAnalyser {
public:
    int NUM_BARK_BANDS = 24;
    maxiBarkScaleAnalyser() {}
    ~maxiBarkScaleAnalyser() { if (h_) mxb_bark_destroy(h_); if (ctx_) mxb_ctx_destroy(ctx_); }
    maxiBarkScaleAnalyser(const maxiBarkScaleAnalyser&) = delete;
    /* device: where the analyser computes when it is not fused into a 1024-point transform */
    void setup(unsigned int sR, unsigned int bS, int device = 0) {
        if (h_) { mxb_bark_destroy(h_); h_ = nullptr; }
        sampleRate_ = sR; bufferSize_ = bS; device_ = device; isSetup_ = true;
    }
    inline double* specificLoudness(const float* normalisedSpectrum);
    inline double* relativeLoudness(const float* normalisedSpectrum);
    inline double* totalLoudness(const float* normalisedSpectrum);
    const double* specificLoudnessOf(int channel, int frame) const { return spec_.data() + ((size_t)channel * (size_t)maxf_ + (size_t)frame) * 24; }
    const double* relativeLoudnessOf(int channel, int frame) const { return rel_.data() + ((size_t)channel * (size_t)maxf_ + (size_t)frame) * 24; }
    double totalLoudnessOf(int channel, int frame) const { return tot_[(size_t)channel * (size_t)maxf_ + (size_t)frame]; }
private:
    friend class maxiFFT;
    inline void own(const float* spectrum, const char* who);
    mxb_bark* handle() {
        using maxib200_detail::check;
        if (!h_) {
            if (!ctx_) check(mxb_ctx_create(device_, (int32_t)maxiSettings::sampleRate, &ctx_), "mxb_ctx_create");
            check(mxb_bark_create(ctx_, (int32_t)sampleRate_, (int32_t)bufferSize_, &h_), "mxb_bark_create");
        }
        return h_;
    }
    maxiFFT* fft_ = nullptr;
    mxb_ctx* ctx_ = nullptr;
    mxb_bark* h_ = nullptr;
    unsigned int sampleRate_ = 0, bufferSize_ = 0;
    bool isSetup_ = false;
    int device_ = 0, maxf_ = 0, last_ = -1;
    std::vector<float> rows_;                               /* the fired frames of a block, packed for mxb_bark_process */
    std::vector<double> spec_, rel_, tot_;
};
typedef maxiBarkScaleAnalyser<double> maxiBark;

/* maxiFFT, src/libs/maxiFFT.h:46-120: process() takes one block of samples per channel, or -- the reference's signature, for a
 * single channel -- one sample */
class maxiFFT {
public:
    enum fftModes { NO_POLAR_CONVERSION = 0, WITH_POLAR_CONVERSION = 1 };
    explicit maxiFFT(int channels = 1, int device = 0) : C_(channels), device_(device) {}
    ~maxiFFT() { if (h_) mxb_stft_destroy(h_); if (ctx_) mxb_ctx_destroy(ctx_); }
    maxiFFT(const maxiFFT&) = delete;
    void setup(int fftSize = 1024, int hopSize = 512, int windowSize = 0) {
        using maxib200_detail::check;
        if (windowSize > fftSize) throw maxiError(MXB_ERR_INVALID, "maxiFFT::setup: windowSize > fftSize overflows the reference's buffer (maxiFFT.cpp:48-51); rejected");
        check(mxb_ctx_create(device_, (int32_t)maxiSettings::sampleRate, &ctx_), "mxb_ctx_create");
        check(mxb_stft_create(ctx_, C_, fftSize, hopSize, &h_), "mxb_stft_create");
        fftSize_ = fftSize; hop_ = hopSize; bins_ = fftSize / 2;
        /* the reference's magnitudes / phases exist (as zeros) before the first frame: a patch may hand them to maxiIFFT at once */
        mags_.assign((size_t)C_ * (size_t)bins_, 0.f); phases_.assign((size_t)C_ * (size_t)bins_, 0.f); maxf_ = 1;
        hopbuf_.clear(); hopbuf_.reserve((size_t)hop_);
        if (oct_) oct_->create();
    }
    /* bool process(float value, fftModes mode), src/libs/maxiFFT.cpp:65-91 -- the reference's per-sample signature, for a transform of
     * ONE channel: the samples of a hop are collected on the host (no arithmetic) and handed over together; true on the sample that
     * completes a frame, exactly where the reference returns it (the first frame fires after hopSize samples, maxiFFT.cpp:55). Afterwards
     * getMagnitudes() / getPhases() hold that frame's numBins values, as in the reference. */
    bool process(float value, fftModes mode = WITH_POLAR_CONVERSION) {
        if (C_ != 1) throw maxiError(MXB_ERR_INVALID, "maxiFFT::process(float): one sample per call feeds a transform of one channel; use process(values, nSamples)");
        if (!h_) throw maxiError(MXB_ERR_STATE, "maxiFFT::process before setup()");
        hopbuf_.push_back(value);
        if ((int)hopbuf_.size() < hop_) return false;
        const bool fired = process(hopbuf_.data(), hop_, mode, 1);
        hopbuf_.clear();
        return fired;
    }
    /* the spectral analysers of the reference, run by process() on every fired frame: fused into the transform's kernel at fft size
     * 1024, on the magnitudes it wrote at other sizes */
    void attach(maxiFFTOctaveAnalyzer& o) { oct_ = &o; o.fft_ = this; if (h_) o.create(); }
    void attach(maxiBark& b) { bark_ = &b; b.fft_ = this; }
    /* magnitudes of frame f (of the last call) of channel c */
    const float* magnitudesOf(int channel, int frame) const { return mags_.data() + ((size_t)channel * (size_t)maxf_ + (size_t)frame) * (size_t)bins_; }
    mxb_ctx* context() { return ctx_; }
    int channels() const { return C_; }
    /* values: planar [channels][nSamples] (host). Returns true when at least one new frame fired (the reference
     * returns true on the sample that completes a frame); frames() tells how many per channel. maxFrames: rows per channel of the
     * result arrays (0 = enough for any nSamples). */
    bool process(const float* values, int nSamples, fftModes mode = WITH_POLAR_CONVERSION, int maxFrames = 0) {
        return run(values, nSamples, nullptr, mode, maxFrames);
    }
    /* channels that advance independently, as separate maxiFFT objects do: channel c takes nSamples[c] samples (host array [channels]) of
     * values, planar at a row pitch of the largest count, and fires its own frames; frames(c) tells how many. The attached analysers run
     * on each channel's own frames: fused at fft size 1024; at other sizes the Bark analyser gets the fired frames packed, while the
     * octave analyser (state per channel, advanced by whole calls of mxb_octave_process) needs every channel to fire as many frames as
     * the others and throws MXB_ERR_UNSUPPORTED, before anything runs, when they would not. Returns true when any channel fired. */
    bool process(const float* values, const int* nSamples, fftModes mode = WITH_POLAR_CONVERSION, int maxFrames = 0) {
        if (!nSamples) throw maxiError(MXB_ERR_INVALID, "maxiFFT::process: nSamples is NULL");
        return run(values, 0, nSamples, mode, maxFrames);
    }
    int frames() const { return frames_; }             /* the most frames any channel fired in the last call */
    int frames(int channel) const { return framesC_.empty() ? 0 : framesC_[(size_t)channel]; }
    int frameStride() const { return maxf_; }     /* frame f of channel c starts at ((c*frameStride()) + f)*getNumBins() */
    std::vector<float>& getMagnitudes() { return mags_; }
    std::vector<float>& getPhases() { return phases_; }
    /* the spectral post-processors (src/libs/maxiFFT.cpp:101-132), computed by the same kernel while the magnitudes are on chip */
    std::vector<float>& magsToDB() { return magsdb_; }                 /* laid out like getMagnitudes() */
    std::vector<float>& getMagnitudesDB() { return magsdb_; }
    std::vector<float>& spectralFlatness() { return flatness_; }       /* frame f of channel c at c*frameStride() + f */
    std::vector<float>& spectralCentroid() { return centroid_; }
    float* getReal() { return re_.data(); }
    float* getImag() { return im_.data(); }
    int getNumBins() { return bins_; }
    int getFFTSize() { return fftSize_; }
    int getHopSize() { return hop_; }
    int getWindowSize() { return fftSize_; }
private:
    /* one block: every channel nSamples samples (counts NULL), or channel c counts[c] */
    bool run(const float* values, int nSamples, const int* counts, fftModes mode, int maxFrames) {
        if (!h_) throw maxiError(MXB_ERR_STATE, "maxiFFT::process before setup()");
        std::vector<int32_t> cnt, expect;
        if (counts) {
            cnt.assign(counts, counts + C_);
            nSamples = 0;
            for (int32_t k : cnt) nSamples = k > nSamples ? k : nSamples;           /* the row pitch */
        }
        const int maxf = maxFrames > 0 ? maxFrames : nSamples / hop_ + 2;
        const size_t len = (size_t)C_ * (size_t)maxf * (size_t)bins_;
        const bool polar = mode == WITH_POLAR_CONVERSION;
        re_.resize(len); im_.resize(len);
        if (polar) {
            mags_.resize(len); phases_.resize(len); magsdb_.resize(len);
            flatness_.assign((size_t)C_ * (size_t)maxf, 0.f); centroid_.assign((size_t)C_ * (size_t)maxf, 0.f);
        }
        mxb_stft_outputs o;
        o.mags = polar ? mags_.data() : nullptr; o.phases = polar ? phases_.data() : nullptr;
        o.re = re_.data(); o.im = im_.data();
        o.mags_db = polar ? magsdb_.data() : nullptr;
        o.flatness = polar ? flatness_.data() : nullptr; o.centroid = polar ? centroid_.data() : nullptr;
        o.coeffs = nullptr;
        int32_t nf = 0;
        const bool post = polar && ((oct_ && oct_->h_) || bark_);
        if (!polar && (oct_ || bark_)) throw maxiError(MXB_ERR_INVALID, "maxiFFT::process: the attached analysers read magnitudes (WITH_POLAR_CONVERSION)");
        mxb_stft_post q;
        std::memset(&q, 0, sizeof(q));
        if (post) {
            if (oct_ && oct_->h_) {
                maxiFFTOctaveAnalyzer& a = *oct_;
                if (a.nSpectrum != bins_)
                    throw maxiError(MXB_ERR_INVALID, "maxiFFT::process: the attached maxiFFTOctaveAnalyzer was set up for " + std::to_string(a.nSpectrum) +
                                                     " bands; the transform has " + std::to_string(bins_) + " bins");
                maxib200_detail::check(mxb_octave_config(a.h_, a.peakHoldTime, a.peakDecayRate, a.linearEQIntercept, a.linearEQSlope), "mxb_octave_config");
                const size_t na = (size_t)C_ * (size_t)maxf * (size_t)(a.nAverages > 0 ? a.nAverages : 1);
                a.avg_.resize(na); a.pk_.resize(na); a.maxf_ = maxf;
                q.octave = a.h_; q.octave_averages = a.avg_.data(); q.octave_peaks = a.pk_.data();
            }
            if (bark_) {
                maxiBark& b = *bark_;
                if (!b.isSetup_) throw maxiError(MXB_ERR_STATE, "maxiBark attached but never setup()");
                if (b.sampleRate_ != (unsigned)maxiSettings::sampleRate || b.bufferSize_ != (unsigned)fftSize_)
                    throw maxiError(MXB_ERR_UNSUPPORTED, "maxiBark::setup(sR, bS) must name the attached transform's sample rate and fft size");
                const size_t nb = (size_t)C_ * (size_t)maxf;
                b.spec_.resize(nb * 24); b.rel_.resize(nb * 24); b.tot_.resize(nb); b.maxf_ = maxf;
                q.bark = 1; q.bark_specific = b.spec_.data(); q.bark_relative = b.rel_.data(); q.bark_total = b.tot_.data();
            }
        }
        const bool fused = post && fftSize_ == 1024;          /* the 1024-point kernel computes the analysers itself */
        if (counts && q.octave && !fused) {
            /* the frames each channel will fire, from its position: mxb_octave_process advances every channel by the same count */
            std::vector<int32_t> pos((size_t)C_);
            maxib200_detail::check(mxb_stft_get_pos(h_, pos.data()), "mxb_stft_get_pos");
            int first = -1;
            for (int c = 0; c < C_; ++c) {
                const long long a = (long long)pos[(size_t)c] + cnt[(size_t)c];
                const int f = a >= fftSize_ ? (int)((a - fftSize_) / hop_) + 1 : 0;
                if (c == 0) first = f;
                else if (f != first)
                    throw maxiError(MXB_ERR_UNSUPPORTED, "maxiFFT::process: an attached maxiFFTOctaveAnalyzer needs every channel to fire as many frames "
                                                         "as the others at fft size " + std::to_string(fftSize_) + " (fused per channel at 1024 only)");
            }
        }
        framesC_.assign((size_t)C_, 0);
        if (counts) {
            maxib200_detail::check(mxb_stft_process_ragged(h_, values, nSamples, 1, cnt.data(), maxf, &o, fused ? &q : nullptr, nullptr, framesC_.data(),
                                                           MXB_MEM_HOST, nullptr), "mxb_stft_process_ragged");
            for (int32_t f : framesC_) nf = f > nf ? f : nf;
        } else if (fused) {
            maxib200_detail::check(mxb_stft_process3(h_, values, nSamples, 1, nSamples, maxf, &o, &q, nullptr, &nf, MXB_MEM_HOST, nullptr),
                                   "mxb_stft_process3");
        } else {
            maxib200_detail::check(mxb_stft_process2(h_, values, nSamples, 1, nSamples, maxf, &o, nullptr, &nf, MXB_MEM_HOST, nullptr),
                                   "mxb_stft_process2");
        }
        if (!counts) framesC_.assign((size_t)C_, nf);
        if (post && !fused && nf > 0) {
            /* frames 0 .. nf - 1 of every channel, in order (the same count for every channel: checked above) */
            if (q.octave)
                maxib200_detail::check(mxb_octave_process(q.octave, mags_.data(), nf, maxf, q.octave_averages, q.octave_peaks, MXB_MEM_HOST, nullptr),
                                       "mxb_octave_process");
            if (q.bark) runBark(maxf);
        }
        frames_ = nf; maxf_ = maxf;
        const int f0 = framesC_[0];
        if (oct_ && oct_->h_ && f0 > 0) { oct_->averages = const_cast<float*>(oct_->averagesOf(0, f0 - 1)); oct_->peaks = const_cast<float*>(oct_->peaksOf(0, f0 - 1)); }
        if (bark_) bark_->last_ = f0 > 0 ? f0 - 1 : -1;
        return nf > 0;
    }
    /* Bark on the fired frames of every channel (frames(c) of channel c): in place when they are contiguous in the [C][maxf] layout, else
     * packed into one call and the results put back at their rows */
    void runBark(int maxf) {
        maxiBark& b = *bark_;
        size_t n = 0;
        bool whole = true;
        for (int c = 0; c < C_; ++c) { n += (size_t)framesC_[(size_t)c]; whole = whole && (framesC_[(size_t)c] == maxf || c == C_ - 1); }
        const size_t bins = (size_t)bins_;
        if (n == 0) return;
        if (whole && (C_ == 1 || framesC_[0] == maxf)) {
            maxib200_detail::check(mxb_bark_process(b.handle(), mags_.data(), (int64_t)n, b.spec_.data(), b.rel_.data(), b.tot_.data(), MXB_MEM_HOST, nullptr),
                                   "mxb_bark_process");
            return;
        }
        b.rows_.resize(n * bins);
        for (size_t c = 0, k = 0; c < (size_t)C_; k += (size_t)framesC_[c], ++c)
            std::memcpy(&b.rows_[k * bins], &mags_[c * maxf * bins], sizeof(float) * framesC_[c] * bins);
        std::vector<double> sp(n * 24), rl(n * 24), tt(n);
        maxib200_detail::check(mxb_bark_process(b.handle(), b.rows_.data(), (int64_t)n, sp.data(), rl.data(), tt.data(), MXB_MEM_HOST, nullptr),
                               "mxb_bark_process");
        for (size_t c = 0, k = 0; c < (size_t)C_; k += (size_t)framesC_[c], ++c) {
            const size_t dst = c * (size_t)maxf, nfc = (size_t)framesC_[c];
            std::memcpy(&b.spec_[dst * 24], &sp[k * 24], sizeof(double) * 24 * nfc);
            std::memcpy(&b.rel_[dst * 24], &rl[k * 24], sizeof(double) * 24 * nfc);
            std::memcpy(&b.tot_[dst], &tt[k], sizeof(double) * nfc);
        }
    }
    int C_, device_;
    mxb_ctx* ctx_ = nullptr; mxb_stft* h_ = nullptr;
    int fftSize_ = 0, hop_ = 0, bins_ = 0, frames_ = 0, maxf_ = 0;
    std::vector<int32_t> framesC_;                          /* frames each channel fired in the last call */
    std::vector<float> mags_, phases_, re_, im_, magsdb_, flatness_, centroid_, hopbuf_;
    maxiFFTOctaveAnalyzer* oct_ = nullptr;
    maxiBark* bark_ = nullptr;
};

inline void maxiFFTOctaveAnalyzer::create() {
    using maxib200_detail::check;
    if (!isSetup_ || (fft_ && !fft_->context())) return;
    if (h_) { mxb_octave_destroy(h_); h_ = nullptr; }
    if (!fft_ && !ctx_) check(mxb_ctx_create(device_, (int32_t)maxiSettings::sampleRate, &ctx_), "mxb_ctx_create");
    check(mxb_octave_create(fft_ ? fft_->context() : ctx_, fft_ ? fft_->channels() : 1, samplingRate, nSpectrum, nAveragesPerOctave, &h_), "mxb_octave_create");
    nAverages = mxb_octave_n_averages(h_);
    if (!fft_) {      /* the results of calculate(): one frame of one channel */
        avg_.assign((size_t)nAverages, 0.f); pk_.assign((size_t)nAverages, 0.f); maxf_ = 1;
        averages = avg_.data(); peaks = pk_.data();
    }
}
inline void maxiFFTOctaveAnalyzer::calculate(const float* fftData) {
    using maxib200_detail::check;
    if (!fft_) {
        if (!h_) throw maxiError(MXB_ERR_STATE, "maxiFFTOctaveAnalyzer::calculate before setup()");
        check(mxb_octave_config(h_, peakHoldTime, peakDecayRate, linearEQIntercept, linearEQSlope), "mxb_octave_config");
        check(mxb_octave_process(h_, fftData, 1, 1, avg_.data(), pk_.data(), MXB_MEM_HOST, nullptr), "mxb_octave_process");
        averages = avg_.data(); peaks = pk_.data();
        return;
    }
    if (!h_ || fft_->frames() <= 0) throw maxiError(MXB_ERR_STATE, "maxiFFTOctaveAnalyzer::calculate: the attached maxiFFT has fired no frame; its process() runs the analyser per frame");
    if (fftData != fft_->magnitudesOf(0, fft_->frames() - 1) && fftData != fft_->magnitudesOf(0, 0))
        throw maxiError(MXB_ERR_UNSUPPORTED, "maxiFFTOctaveAnalyzer::calculate: an attached analyser has analysed its transform's frame already; only those magnitudes can be passed");
}
template <class T> inline void maxiBarkScaleAnalyser<T>::own(const float* spectrum, const char* who) {
    if (!fft_) {      /* not attached: analyse the spectrum handed in */
        if (!isSetup_) throw maxiError(MXB_ERR_STATE, std::string(who) + " before setup()");
        spec_.resize(24); rel_.resize(24); tot_.resize(1); maxf_ = 1; last_ = 0;
        maxib200_detail::check(mxb_bark_process(handle(), spectrum, 1, spec_.data(), rel_.data(), tot_.data(), MXB_MEM_HOST, nullptr), "mxb_bark_process");
        return;
    }
    if (last_ < 0) throw maxiError(MXB_ERR_STATE, std::string(who) + ": the attached maxiFFT has fired no frame; its process() runs the analyser per frame");
    if (spectrum != fft_->magnitudesOf(0, last_) && spectrum != fft_->magnitudesOf(0, 0))
        throw maxiError(MXB_ERR_UNSUPPORTED, std::string(who) + ": only the attached transform's own magnitudes can be analysed");
}
template <class T> inline double* maxiBarkScaleAnalyser<T>::specificLoudness(const float* sp) { own(sp, "maxiBark::specificLoudness"); return const_cast<double*>(specificLoudnessOf(0, last_)); }
template <class T> inline double* maxiBarkScaleAnalyser<T>::relativeLoudness(const float* sp) { own(sp, "maxiBark::relativeLoudness"); return const_cast<double*>(relativeLoudnessOf(0, last_)); }
template <class T> inline double* maxiBarkScaleAnalyser<T>::totalLoudness(const float* sp) { own(sp, "maxiBark::totalLoudness"); return &tot_[(size_t)last_]; }

/* maxiIFFT (SPECTRUM mode), src/libs/maxiFFT.h:125-156; COMPLEX mode yields zeros in the reference on Linux and is not offered */
class maxiIFFT {
public:
    enum fftModes { SPECTRUM = 0 };
    explicit maxiIFFT(int channels = 1, int device = 0) : C_(channels), device_(device) {}
    ~maxiIFFT() { if (h_) mxb_istft_destroy(h_); if (ctx_) mxb_ctx_destroy(ctx_); }
    maxiIFFT(const maxiIFFT&) = delete;
    /* fftSize: a power of two from 64 to 2048, hopSize: 1 to fftSize -- every spectrum maxiFFT produces can be resynthesised */
    void setup(int fftSize = 1024, int hopSize = 512, int windowSize = 0) {
        using maxib200_detail::check;
        /* the reference windows with genWindow(3, windowSize ? windowSize : fftSize) (maxiFFT.cpp:141-152): another size is another window */
        if (windowSize != 0 && windowSize != fftSize) throw maxiError(MXB_ERR_UNSUPPORTED, "maxiIFFT::setup: windowSize must be 0 or fftSize");
        check(mxb_ctx_create(device_, (int32_t)maxiSettings::sampleRate, &ctx_), "mxb_ctx_create");
        check(mxb_istft_create(ctx_, C_, fftSize, hopSize, &h_), "mxb_istft_create");
        hop_ = hopSize; bins_ = fftSize / 2;
    }
    /* data1/data2: magnitudes / phases, frame f of channel c at (c*frames + f)*bins; returns planar [channels][frames*hop] */
    std::vector<float>& process(const std::vector<float>& data1, const std::vector<float>& data2, int frames, fftModes = SPECTRUM) {
        out_.resize((size_t)C_ * (size_t)frames * (size_t)hop_);
        maxib200_detail::check(mxb_istft_process(h_, data1.data(), data2.data(), frames, out_.data(), MXB_MEM_HOST, nullptr), "mxb_istft_process");
        return out_;
    }
    /* channels that advance independently, as separate maxiIFFT objects do: channel c resynthesises frames[c] frames (host array
     * [channels], 0 .. maxFrames) of data1 / data2, frame f of channel c at (c*maxFrames + f)*bins; returns planar [channels][maxFrames*hop],
     * channel c's first frames[c]*hop samples its output. A channel with no frame keeps its overlap-add buffer. */
    std::vector<float>& process(const std::vector<float>& data1, const std::vector<float>& data2, const int* frames, int maxFrames, fftModes = SPECTRUM) {
        if (!frames) throw maxiError(MXB_ERR_INVALID, "maxiIFFT::process: frames is NULL");
        const size_t need = (size_t)C_ * (size_t)(maxFrames > 0 ? maxFrames : 0) * (size_t)bins_;
        if (data1.size() < need || data2.size() < need) throw maxiError(MXB_ERR_INVALID, "maxiIFFT::process: magnitudes / phases shorter than channels x maxFrames x numBins");
        const std::vector<int32_t> fr(frames, frames + C_);
        out_.assign((size_t)C_ * (size_t)(maxFrames > 0 ? maxFrames : 0) * (size_t)hop_, 0.f);
        maxib200_detail::check(mxb_istft_process_ragged(h_, data1.data(), data2.data(), fr.data(), maxFrames, out_.data(), MXB_MEM_HOST, nullptr),
                               "mxb_istft_process_ragged");
        return out_;
    }
    /* float process(mags, phases, mode), src/libs/maxiFFT.cpp:154-192 -- the reference's per-sample signature, for ONE channel: the spectrum is
     * read on the first call of every hop (pos == 0, like the reference), that frame is resynthesised and overlap-added on the device, and its
     * hop samples are handed out one per call. */
    float process(std::vector<float>& mags, std::vector<float>& phases, fftModes = SPECTRUM) {
        if (C_ != 1) throw maxiError(MXB_ERR_INVALID, "maxiIFFT::process per sample feeds one channel; use process(mags, phases, frames)");
        if (!h_) throw maxiError(MXB_ERR_STATE, "maxiIFFT::process before setup()");
        if (pos_ == 0) {
            if ((int)mags.size() < bins_ || (int)phases.size() < bins_) throw maxiError(MXB_ERR_INVALID, "maxiIFFT::process: magnitudes / phases shorter than numBins");
            cur_.resize((size_t)hop_);
            maxib200_detail::check(mxb_istft_process(h_, mags.data(), phases.data(), 1, cur_.data(), MXB_MEM_HOST, nullptr), "mxb_istft_process");
        }
        const float v = cur_[(size_t)pos_];
        if (++pos_ == hop_) pos_ = 0;
        return v;
    }
    int getNumBins() { return bins_; }
private:
    int C_, device_;
    mxb_ctx* ctx_ = nullptr; mxb_istft* h_ = nullptr; int hop_ = 0, bins_ = 0, pos_ = 0;
    std::vector<float> out_, cur_;
};

#endif /* MAXIMILIAN_B200_HPP */
