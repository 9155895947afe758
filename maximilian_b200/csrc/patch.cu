// Voice patches: a per-voice signal graph -- the body of any reference play() built from the stages of maxib200.h --
// run sample by sample for V voices by one interpreting kernel (K8).
//
// The fused bank kernels (K1 / K2) are hard-wired to oscillator -> envelope -> filter -> delay -> mix, the chains
// BASELINE.json measures. Real patches are graphs: two oscillators summed into one filter, an LFO added to a frequency,
// an envelope multiplying the filter OUTPUT (cpp/commandline/maximilian_examples/15.polysynth/main.cpp:54-70), a trigger
// that changes on any sample (10.Filters/main.cpp:27-36). A patch is a short list of stages over 16 per-voice registers;
// operands are registers, per-voice parameter arrays, scalar constants or per-sample input streams. Every voice runs the
// SAME program, so the interpreter's dispatch is warp-uniform (no divergence): one thread = one voice, registers /
// parameters / stage state live in shared memory for the block ([slot][thread], conflict-free), loaded from and stored
// to SoA arrays in HBM once per block like the fused kernels do.
//
// Each stage body is the reference method restated (same statements, same order, -fmad=false). Stages whose reference
// method designs coefficients from its arguments on every call (lores/hires/bandpass, maxiSVF::setParams, maxiBiquad::set,
// pow/atan in maxiNonlinearity, pow in maxiEnvGen) call libdevice where the reference calls glibc: 1e-9 relative instead
// of bit-identical; everything else is bit-identical.
#include <math.h>

#include <new>

#include "patch_impl.cuh"
#include "exchange.cuh"

using namespace mxb;

namespace {

// MULTI_EG: the patch plays more than one maxiEnvGen shape. With one shape every ENVGEN stage plays shape 0, whose table and flags are then
// read at fixed offsets of the argument block: a shape index read at run time makes ptxas spill in the stage loop, which cost the interpreter
// about 2 % on the polysynth patch (H100 80GB HBM3, 700 W), a patch without any maxiEnvGen stage.
// EVENTS: the patch has MXB_IN_EVENTS streams. Each keeps three words per voice in shared memory after the state -- its held value,
// the cursor into this call's events and the frame of the event at the cursor -- advanced once per sample before the stage loop. A patch
// without events streams runs the instantiation that has none of it: the same code, launch shape and shared-memory layout as before.
template <bool MULTI_EG, bool EVENTS>
__global__ void __launch_bounds__(kPatchThreads) patch_kernel(const PatchArgs a) {
    extern __shared__ double psm[];
    __shared__ mxb_stage s_stage[kMaxStages];
    __shared__ int s_sbase[kMaxStages], s_ring[kMaxStages];
    __shared__ double s_const[kMaxConsts];
    for (int i = threadIdx.x; i < a.n_stages; i += blockDim.x) { s_stage[i] = a.stages[i]; s_sbase[i] = a.state_base[i]; s_ring[i] = a.ring_of[i]; }
    for (int i = threadIdx.x; i < kMaxConsts; i += blockDim.x) s_const[i] = a.consts[i];
    const int tid = threadIdx.x, lane = tid & 31;
    const long long v = (long long)blockIdx.x * blockDim.x + tid;
    const bool live = v < a.V;
    const size_t V = (size_t)a.V, vv = live ? (size_t)v : 0;
    const Lane reg{psm + tid, kPatchThreads};
    const Lane par{psm + (size_t)kMaxRegs * kPatchThreads + tid, kPatchThreads};
    const Lane st{psm + (size_t)(kMaxRegs + a.n_params) * kPatchThreads + tid, kPatchThreads};
    for (int i = 0; i < kMaxRegs; ++i) reg[i] = 0.0;
    for (int i = 0; i < a.n_params; ++i) par[i] = a.params[(size_t)i * V + vv];
    for (int i = 0; i < a.n_state; ++i) st[i] = a.state[(size_t)i * V + vv];
    const Lane evl{psm + (size_t)(kMaxRegs + a.n_params + a.n_state) * kPatchThreads + tid, kPatchThreads};      // 3 words per events stream
    if (EVENTS)
        for (int e = 0; e < a.n_ev; ++e) {
            evl[3 * e] = a.held[(size_t)e * V + vv];
            ev_start(a.ev[e], vv, live, evl[3 * e + 1], evl[3 * e + 2]);
        }
    __syncthreads();
    const int gwarp = (int)(((long long)blockIdx.x * blockDim.x + tid) >> 5);
    const double sr = a.sr;

    for (int t = 0; t < a.n_frames; ++t) {
        double ml = 0.0, mr = 0.0;
        for (int i = 0; i < kMaxRegs; ++i) reg[i] = 0.0;          // registers read 0 until a stage of this sample writes them
        if (EVENTS)
            for (int e = 0; e < a.n_ev; ++e) ev_advance(a.ev[e], vv, t, evl[3 * e], evl[3 * e + 1], evl[3 * e + 2]);
        auto fetch = [&](const int src) -> double {
            if (src < 0) return 0.0;
            const int k = src & 0xff;
            switch (src >> 8) {
                case 0: return reg[k];
                case 1: return par[k];
                case 2: return s_const[k];
                default:
                    if (EVENTS && a.in_kind[k] == MXB_IN_EVENTS) return evl[3 * a.ev_of[k]];
                    return live ? patch_input(a, k, (size_t)t, vv, V) : 0.0;
            }
        };
        for (int si = 0; si < a.n_stages; ++si) {
            const mxb_stage& g = s_stage[si];
            const int sb = s_sbase[si];
            double y = 0.0;
            switch (g.op) {
                case MXB_OP_OSC: {
                    OscRegs o; osc_state<true>(st, sb, o);
                    y = stage_osc(g.kind, o.phase, o.output, fetch(g.src[0]), fetch(g.src[1]), fetch(g.src[2]), sr, a.sine, a.transition, a.sine_before);
                    osc_state<false>(st, sb, o);
                    break;
                }
                case MXB_OP_ENV_ADSR:
                case MXB_OP_ENV_AR: {
                    PatchEnvRegs e; env_state<true>(st, sb, e);
                    const double in = fetch(g.src[0]);
                    const bool trig = trigger_arg(fetch(g.src[1]));
                    if (g.op == MXB_OP_ENV_ADSR) {
                        e.att = fetch(g.src[2]); e.dec = fetch(g.src[3]); e.sus = fetch(g.src[4]); e.rel = fetch(g.src[5]);
                        e.holdtime = env_holdtime<PatchEnvRegs>(fetch(g.src[6]));
                        y = env_tick(e, in, trig);
                    } else {
                        e.att = fetch(g.src[2]); e.rel = fetch(g.src[3]); e.holdtime = env_holdtime<PatchEnvRegs>(fetch(g.src[4]));
                        e.dec = 0.0; e.sus = 0.0;
                        y = env_ar_tick(e, in, trig);
                    }
                    env_state<false>(st, sb, e);
                    break;
                }
                case MXB_OP_ENVGEN: {
                    EgRegs q; envgen_state<true>(st, sb, q);
                    const int k = MULTI_EG ? g.kind : 0;
                    y = envgen_tick(q, fetch(g.src[0]), a.eg[k], a.eg_n[k], a.eg_loop[k], a.eg_retrigger[k]);
                    envgen_state<false>(st, sb, q);
                    break;
                }
                case MXB_OP_FILTER: {
                    const double in = fetch(g.src[0]);
                    FiltRegs f;
                    if (g.kind == MXB_FILT_LORES || g.kind == MXB_FILT_HIRES) {
                        filt_state<2, true>(st, sb, f);
                        filt_design<FILT_T_LORES>(f, fetch(g.src[1]), fetch(g.src[2]), sr);
                        y = g.kind == MXB_FILT_LORES ? filt_tick<FILT_T_LORES>(f, in, nullptr) : filt_tick<FILT_T_HIRES>(f, in, nullptr);
                        filt_state<2, false>(st, sb, f);
                    } else if (g.kind == MXB_FILT_LOPASS || g.kind == MXB_FILT_HIPASS) {
                        filt_state<1, true>(st, sb, f);
                        y = onepole_tick(g.kind, f.s0, in, fetch(g.src[1]));
                        filt_state<1, false>(st, sb, f);
                    } else {
                        filt_state<2, true>(st, sb, f);
                        double c0, c1, c2;
                        design_bandpass(fetch(g.src[1]), fetch(g.src[2]), sr, c0, c1, c2);
                        y = bandpass_tick(f.s0, f.s1, in, c0, c1, c2);
                        filt_state<2, false>(st, sb, f);
                    }
                    break;
                }
                case MXB_OP_SVF: {
                    FiltRegs f; filt_state<3, true>(st, sb, f);
                    filt_design<FILT_T_SVF>(f, fetch(g.src[1]), fetch(g.src[2]), sr);
                    const double mixw[4] = {fetch(g.src[3]), fetch(g.src[4]), fetch(g.src[5]), fetch(g.src[6])};
                    y = filt_tick<FILT_T_SVF>(f, fetch(g.src[0]), mixw);
                    filt_state<3, false>(st, sb, f);
                    break;
                }
                case MXB_OP_BIQUAD: {
                    FiltRegs f; filt_state<2, true>(st, sb, f);
                    double cf[5];
                    design_biquad_one(g.kind, fetch(g.src[1]), fetch(g.src[2]), fetch(g.src[3]), sr, cf);
                    f.c0 = cf[0]; f.c1 = cf[1]; f.c2 = cf[2]; f.c3 = cf[3]; f.c4 = cf[4];
                    y = filt_tick<FILT_T_BIQUAD>(f, fetch(g.src[0]), nullptr);
                    filt_state<2, false>(st, sb, f);
                    break;
                }
                case MXB_OP_DCBLOCK: {
                    FiltRegs f; filt_state<2, true>(st, sb, f);
                    y = dcblock_tick(f.s0, f.s1, fetch(g.src[0]), fetch(g.src[1]));
                    filt_state<2, false>(st, sb, f);
                    break;
                }
                case MXB_OP_NONLIN: y = nonlin_eval(g.kind, fetch(g.src[0]), fetch(g.src[1]), fetch(g.src[2])); break;
                case MXB_OP_DELAY:
                case MXB_OP_FLANGER: {
                    double* ring = a.rings + (size_t)s_ring[si] * (size_t)a.taps * V + vv;      // slot r of this voice at ring[r * V]
                    const double in = fetch(g.src[0]);
                    int ph; delay_state<true>(st, sb, ph);
                    if (g.op == MXB_OP_DELAY) {
                        const int size = int_arg(fetch(g.src[1]));
                        const double fb = fetch(g.src[2]);
                        const bool fp = g.kind == MXB_DELAY_FROM_POSITION;
                        y = delay_tick(fp, ring, V, a.taps, live, ph, in, size, fb, fp ? int_arg(fetch(g.src[3])) : 0);
                    } else {
                        OscRegs lfo; osc_state<true>(st, sb + 1, lfo);
                        const unsigned int delay = uint_arg(fetch(g.src[1]));
                        const double fb = fetch(g.src[2]);
                        y = flanger_tick(ring, V, a.taps, live, ph, lfo.phase, lfo.output, in, delay, fb, fetch(g.src[3]), fetch(g.src[4]), sr);
                        osc_state<false>(st, sb + 1, lfo);
                    }
                    delay_state<false>(st, sb, ph);
                    break;
                }
                case MXB_OP_CHORUS: {
                    double* ring = a.rings + (size_t)s_ring[si] * (size_t)a.taps * V + vv;      // this voice's two lines: ring index s_ring[si], + 1
                    int ph1, ph2;
                    FiltRegs lp; chorus_state<true>(st, sb, ph1, ph2, lp);
                    filt_design<FILT_T_LORES>(lp, fetch(g.src[3]), 1.0, sr);
                    y = chorus_tick(ring, ring + (size_t)a.taps * V, V, a.taps, live, ph1, ph2, lp, fetch(g.src[0]), uint_arg(fetch(g.src[1])), fetch(g.src[2]),
                                    fetch(g.src[4]), fetch(g.src[5]));
                    chorus_state<false>(st, sb, ph1, ph2, lp);
                    break;
                }
                case MXB_OP_ADD: y = fetch(g.src[0]) + fetch(g.src[1]); break;
                case MXB_OP_SUB: y = fetch(g.src[0]) - fetch(g.src[1]); break;
                case MXB_OP_MUL: y = fetch(g.src[0]) * fetch(g.src[1]); break;
                case MXB_OP_DIV: y = fetch(g.src[0]) / fetch(g.src[1]); break;
                case MXB_OP_MIX_STEREO: {        // maxiMix::stereo, src/maximilian.cpp:503-509, accumulated over the stages of this sample
                    const double in = fetch(g.src[0]), x = fetch(g.src[1]);
                    if (live) mix_stereo_acc(ml, mr, in, x);
                    break;
                }
                case MXB_OP_OUT:
                    if (live && a.out) a.out[(size_t)t * V + vv] = fetch(g.src[0]);
                    break;
                default: break;
            }
            if (g.dst >= 0) reg[g.dst] = y;
        }
        if (a.partials) mix_warp_store(ml, mr, lane, a.partials, (size_t)t, (size_t)a.W, (size_t)gwarp);      // the second kernel adds the warps in order
    }
    if (live) for (int i = 0; i < a.n_state; ++i) a.state[(size_t)i * V + (size_t)v] = st[i];
    if (EVENTS && live) for (int e = 0; e < a.n_ev; ++e) a.held[(size_t)e * V + (size_t)v] = evl[3 * e];
}

// MXB_PATCH_MODE=interpret | fused overrides the default (fused) for patches created afterwards: an A/B and debugging hook
int patch_default_mode() {
    const char* e = getenv("MXB_PATCH_MODE");
    if (e && strcmp(e, "interpret") == 0) return MXB_PATCH_INTERPRET;
    return MXB_PATCH_FUSED;
}

bool src_ok(int s, const mxb_patch_desc* d) {
    if (s == MXB_NONE) return true;
    if (s < 0) return false;
    const int k = s & 0xff;
    switch (s >> 8) {
        case 0: return k < kMaxRegs;
        case 1: return k < d->n_params;
        case 2: return k < d->n_consts;
        case 3: return k < d->n_inputs;
        default: return false;
    }
}

// The checks of a stage list that need nothing but the descriptor, shared by mxb_patch_create / create2 and mxb_patch_codegen: a program
// the code generator accepts is one a patch can be created from. ENVGEN kinds index the first `n_shapes` maxiEnvGen shapes.
int validate_stages(const mxb_patch_desc* d, const int n_shapes, const char* who) {
    MXB_REQUIRE(d->n_stages > 0 && d->n_stages <= kMaxStages, MXB_ERR_INVALID, "%s: n_stages %d (1..%d)", who, d->n_stages, kMaxStages);
    MXB_REQUIRE(d->n_params >= 0 && d->n_params <= kMaxParams && d->n_consts >= 0 && d->n_consts <= kMaxConsts && d->n_inputs >= 0 && d->n_inputs <= kMaxInputs,
                MXB_ERR_INVALID, "%s: n_params %d n_consts %d n_inputs %d", who, d->n_params, d->n_consts, d->n_inputs);
    MXB_REQUIRE(d->n_consts == 0 || d->consts, MXB_ERR_INVALID, "%s: consts is NULL", who);
    for (int i = 0; d->input_types && i < d->n_inputs; ++i)
        MXB_REQUIRE(d->input_types[i] >= MXB_IN_F64 && d->input_types[i] <= MXB_IN_EVENTS, MXB_ERR_INVALID, "%s: input_types[%d] = %d", who, i, d->input_types[i]);
    for (int i = 0; i < d->n_stages; ++i) {
        const mxb_stage& g = d->stages[i];
        MXB_REQUIRE(g.op >= MXB_OP_OSC && g.op <= MXB_OP_CHORUS, MXB_ERR_INVALID, "%s: stage %d: unknown op %d", who, i, g.op);
        MXB_REQUIRE(g.dst == MXB_NONE || (g.dst >= 0 && g.dst < kMaxRegs), MXB_ERR_INVALID, "%s: stage %d: dst %d", who, i, g.dst);
        for (int k = 0; k < MXB_STAGE_SRCS; ++k) MXB_REQUIRE(src_ok(g.src[k], d), MXB_ERR_INVALID, "%s: stage %d: operand %d = 0x%x", who, i, k, g.src[k]);
        if (g.op == MXB_OP_OSC) MXB_REQUIRE(g.kind >= MXB_OSC_SINEWAVE && g.kind <= MXB_OSC_SAWN, MXB_ERR_INVALID, "%s: stage %d: osc kind %d", who, i, g.kind);
        if (g.op == MXB_OP_FILTER) MXB_REQUIRE(g.kind == MXB_FILT_LORES || g.kind == MXB_FILT_HIRES || g.kind == MXB_FILT_LOPASS || g.kind == MXB_FILT_HIPASS || g.kind == MXB_FILT_BANDPASS,
                                               MXB_ERR_INVALID, "%s: stage %d: filter kind %d", who, i, g.kind);
        if (g.op == MXB_OP_BIQUAD) MXB_REQUIRE(g.kind >= MXB_BQ_LOWPASS && g.kind <= MXB_BQ_HIGHSHELF, MXB_ERR_INVALID, "%s: stage %d: biquad type %d", who, i, g.kind);
        if (g.op == MXB_OP_NONLIN) MXB_REQUIRE(g.kind >= MXB_NL_ATANDIST && g.kind <= MXB_NL_FASTATAN, MXB_ERR_INVALID, "%s: stage %d: nonlinearity %d", who, i, g.kind);
        if (g.op == MXB_OP_ENVGEN) MXB_REQUIRE(g.kind >= 0 && g.kind < n_shapes, MXB_ERR_INVALID, "%s: stage %d: envelope shape %d of %d", who, i, g.kind, n_shapes);
    }
    return MXB_OK;
}

// maxiEnvGen::setup + setupSegmentTime, src/maximilian.h:2371-2402, 2524-2538: the segment table of one shape from levels / times / curves
void eg_segments(const mxb_envgen_shape& s, const double srd, EgStage* eg) {
    double accumulatedTime = 0;
    for (int i = 0; i < s.stages; ++i) {
        EgStage& e = eg[i];
        e.startlevel = s.levels[i]; e.endlevel = s.levels[i + 1]; e.curve = s.curves[i]; e.pad = 0;
        const double stageTime = s.times[i];
        if (stageTime == MXB_ENVGEN_HOLD) { e.length = 0; e.hold = 1; e.gradient = 0; }
        else {
            const double len = ((stageTime / 1000.0) * srd) + accumulatedTime;
            e.length = (long long)(size_t)floor(len);
            accumulatedTime = len - e.length;
            e.gradient = 1.0 / e.length;
            e.hold = 0;
        }
    }
}

// mxb_patch_create and mxb_patch_create2: `who` names the entry point the caller used in the error messages
int32_t create_patch(mxb_ctx* ctx, const mxb_patch_desc* d, const int32_t n_shapes, const mxb_envgen_shape* shapes, mxb_patch** out, const char* who) {
    MXB_REQUIRE(ctx && d && out && d->stages, MXB_ERR_INVALID, "%s: NULL argument", who);
    *out = nullptr;
    MXB_REQUIRE(d->voices > 0 && d->max_frames > 0, MXB_ERR_INVALID, "%s: voices %d max_frames %d", who, d->voices, d->max_frames);
    MXB_REQUIRE(d->delay_taps >= 0, MXB_ERR_INVALID, "%s: delay_taps %d", who, d->delay_taps);
    MXB_REQUIRE(n_shapes >= 0 && n_shapes <= kMaxEgShapes, MXB_ERR_INVALID, "%s: n_shapes %d (0..%d)", who, n_shapes, kMaxEgShapes);
    MXB_REQUIRE(n_shapes == 0 || shapes, MXB_ERR_INVALID, "%s: shapes is NULL", who);
    for (int k = 0; k < n_shapes; ++k) {
        const mxb_envgen_shape& s = shapes[k];
        MXB_REQUIRE(s.stages >= 0 && s.stages <= kMaxEg, MXB_ERR_INVALID, "%s: shape %d: stages %d (0..%d)", who, k, s.stages, kMaxEg);
        MXB_REQUIRE(s.stages == 0 || (s.levels && s.times && s.curves), MXB_ERR_INVALID, "%s: shape %d needs levels / times / curves", who, k);
        int holds = 0;
        for (int i = 0; i < s.stages; ++i) holds += s.times[i] == MXB_ENVGEN_HOLD;
        MXB_REQUIRE(holds <= 1, MXB_ERR_INVALID, "%s: shape %d has %d HOLD segments (maxiEnvGen::setup allows one)", who, k, holds);
    }
    int rc = validate_stages(d, n_shapes, who);
    if (rc != MXB_OK) return rc;
    int n_state = 0, n_rings = 0;
    bool tables = false;
    for (int i = 0; i < d->n_stages; ++i) {
        const mxb_stage& g = d->stages[i];
        tables = tables || (g.op == MXB_OP_OSC && g.kind >= MXB_OSC_SINEBUF);
        if (patch_stage_rings(g.op)) { MXB_REQUIRE(d->delay_taps > 0, MXB_ERR_INVALID, "%s: stage %d needs delay_taps > 0", who, i); n_rings += patch_stage_rings(g.op); }
        n_state += patch_state_slots(g.op);
    }
    if (tables) MXB_REQUIRE(ctx->d_sine.get(), MXB_ERR_STATE, "%s: sinebuf / sinebuf4 / sawn need the reference's tables: call mxb_ctx_set_tables first", who);
    int n_ev = 0;
    for (int i = 0; d->input_types && i < d->n_inputs; ++i) n_ev += d->input_types[i] == MXB_IN_EVENTS;
    const size_t per_thread = (size_t)(kMaxRegs + d->n_params + n_state + 3 * n_ev);
    MXB_REQUIRE(per_thread * 8 * kPatchThreads <= 200 * 1024, MXB_ERR_UNSUPPORTED,
                "%s: %zu doubles of registers, parameters, state and events streams (3 each) per voice do not fit shared memory", who, per_thread);
    DeviceGuard g(ctx->device);
    std::unique_ptr<mxb_patch> p(new (std::nothrow) mxb_patch());
    MXB_REQUIRE(p, MXB_ERR_ALLOC, "%s: out of host memory", who);
    p->ctx = ctx; p->V = d->voices; p->n_stages = d->n_stages; p->n_params = d->n_params; p->n_consts = d->n_consts; p->n_inputs = d->n_inputs;
    p->max_frames = d->max_frames; p->taps = d->delay_taps; p->n_state = n_state; p->n_rings = n_rings;
    p->stages.assign(d->stages, d->stages + d->n_stages);
    if (d->n_consts) p->consts.assign(d->consts, d->consts + d->n_consts);
    p->mode = patch_default_mode(); p->fused = nullptr; p->ex = nullptr;
    p->n_ev = 0;
    for (int i = 0; i < d->n_inputs; ++i) {
        p->in_type[i] = d->input_types ? d->input_types[i] : MXB_IN_F64;
        p->ev_of[i] = (unsigned char)p->n_ev;
        p->n_ev += p->in_type[i] == MXB_IN_EVENTS;
    }
    int sb = 0, ri = 0;
    for (int i = 0; i < d->n_stages; ++i) {
        p->state_base.push_back(sb); sb += patch_state_slots(p->stages[i].op);
        const int nr = patch_stage_rings(p->stages[i].op);
        p->ring_of.push_back(nr ? ri : -1);
        ri += nr;
    }
    p->n_shapes = n_shapes;
    for (int k = 0; k < n_shapes; ++k) {
        p->eg_n[k] = shapes[k].stages; p->eg_loop[k] = shapes[k].loop; p->eg_retrigger[k] = shapes[k].retrigger;
        eg_segments(shapes[k], (double)(size_t)ctx->sample_rate, p->eg[k]);
    }
    const size_t V = (size_t)p->V;
    if (rc == MXB_OK) rc = p->d_stages.alloc((size_t)d->n_stages);
    if (rc == MXB_OK) rc = p->d_state_base.alloc((size_t)d->n_stages);
    if (rc == MXB_OK) rc = p->d_ring_of.alloc((size_t)d->n_stages);
    if (rc == MXB_OK) rc = p->d_consts.alloc((size_t)kMaxConsts);
    if (rc == MXB_OK) rc = p->params.alloc((size_t)(d->n_params ? d->n_params : 1) * V);
    if (rc == MXB_OK) rc = p->state.alloc((size_t)(n_state ? n_state : 1) * V);
    if (rc == MXB_OK && n_rings) rc = p->rings.alloc((size_t)n_rings * (size_t)p->taps * V);
    if (rc == MXB_OK) rc = p->mix_dev.alloc((size_t)p->max_frames * 2);
    if (rc == MXB_OK && p->n_ev) rc = p->held.alloc((size_t)p->n_ev * V);          // held values start at 0.0
    if (rc != MXB_OK) return rc;
    cudaError_t e = cudaMemcpy(p->d_stages.get(), p->stages.data(), sizeof(mxb_stage) * d->n_stages, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(p->d_state_base.get(), p->state_base.data(), sizeof(int) * d->n_stages, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(p->d_ring_of.get(), p->ring_of.data(), sizeof(int) * d->n_stages, cudaMemcpyHostToDevice);
    if (e == cudaSuccess && d->n_consts) e = cudaMemcpy(p->d_consts.get(), d->consts, sizeof(double) * d->n_consts, cudaMemcpyHostToDevice);
    for (int i = 0; i < d->n_stages && e == cudaSuccess; ++i)
        for (int k = 0; k < patch_state_slots(p->stages[i].op) && e == cudaSuccess; ++k)
            if (patch_state_init(p->stages[i].op, k) != 0.0) {                 // alloc zeroed the others
                const std::vector<double> col(V, patch_state_init(p->stages[i].op, k));
                e = cudaMemcpy(p->state.get() + (size_t)(p->state_base[i] + k) * V, col.data(), sizeof(double) * V, cudaMemcpyHostToDevice);
            }
    if (e != cudaSuccess) { set_error("%s: %s", who, cudaGetErrorString(e)); return MXB_ERR_CUDA; }
    *out = p.release();
    return MXB_OK;
}

// The structural checks of an events descriptor (mxb_events): before any copy or kernel, so that a refused call changes nothing.
// Device-memory arrays are not looked at: whatever they hold, the kernels read voice v's events only inside [first[v], first[v+1]).
int check_events(const mxb_patch* p, const int m, const mxb_events* e, const bool host) {
    MXB_REQUIRE(e->first && e->frame && e->value, MXB_ERR_INVALID, "mxb_patch_process: events stream %d: first / frame / value is NULL", m);
    if (host) {
        MXB_REQUIRE(e->first[0] >= 0, MXB_ERR_INVALID, "mxb_patch_process: events stream %d: first[0] = %d", m, e->first[0]);
        for (int v = 0; v < p->V; ++v)
            MXB_REQUIRE(e->first[v + 1] >= e->first[v], MXB_ERR_INVALID, "mxb_patch_process: events stream %d: first[%d] = %d < first[%d] = %d", m, v + 1,
                        e->first[v + 1], v, e->first[v]);
    }
    return MXB_OK;
}

// the device view of events stream m for this call: host arrays through the patch's staging buffers (first[voices] events)
int stage_events(mxb_patch* p, const int m, const mxb_events* e, const bool host, cudaStream_t s, EvStream* out) {
    const int k = p->ev_of[m];
    const size_t n = host ? (size_t)e->first[p->V] : 0;
    int rc = stage_in(host, e->first, (size_t)p->V + 1, p->ev_first[k], s, &out->first);
    if (rc == MXB_OK) rc = stage_in(host, e->frame, n, p->ev_frame[k], s, &out->frame);
    if (rc == MXB_OK) rc = stage_in(host, e->value, n, p->ev_value[k], s, &out->value);
    return rc;
}

// events stream m's held values ([voices] doubles)
int32_t patch_held_ptr(mxb_patch* p, const int32_t m, double** ptr, const char* who) {
    MXB_REQUIRE(p, MXB_ERR_INVALID, "%s: NULL patch", who);
    MXB_REQUIRE(m >= 0 && m < p->n_inputs && p->in_type[m] == MXB_IN_EVENTS, MXB_ERR_INVALID, "%s: input stream %d is not an events stream", who, m);
    *ptr = p->held.get() + (size_t)p->ev_of[m] * (size_t)p->V;
    return MXB_OK;
}

}  // namespace

extern "C" {

int32_t mxb_ctx_set_tables(mxb_ctx* ctx, const double* sine514, const double* transition1001, double sine_before) {
    MXB_REQUIRE(ctx && sine514 && transition1001, MXB_ERR_INVALID, "mxb_ctx_set_tables: NULL argument");
    DeviceGuard g(ctx->device);
    if (!ctx->d_sine.get()) { int rc = ctx->d_sine.alloc(514 + 1001); if (rc != MXB_OK) return rc; }
    MXB_CUDA(cudaMemcpy(ctx->d_sine.get(), sine514, sizeof(double) * 514, cudaMemcpyHostToDevice));
    MXB_CUDA(cudaMemcpy(ctx->d_sine.get() + 514, transition1001, sizeof(double) * 1001, cudaMemcpyHostToDevice));
    ctx->sine_before = sine_before;
    return MXB_OK;
}

int32_t mxb_patch_create(mxb_ctx* ctx, const mxb_patch_desc* d, mxb_patch** out) {
    MXB_REQUIRE(d, MXB_ERR_INVALID, "mxb_patch_create: NULL argument");
    MXB_REQUIRE(d->eg_stages >= 0 && d->eg_stages <= kMaxEg, MXB_ERR_INVALID, "mxb_patch_create: eg_stages %d (0..%d)", d->eg_stages, kMaxEg);
    bool eg = false;
    for (int i = 0; d->stages && i < d->n_stages && i < kMaxStages; ++i) eg = eg || d->stages[i].op == MXB_OP_ENVGEN;
    if (eg) MXB_REQUIRE(d->eg_stages > 0 && d->eg_levels && d->eg_times && d->eg_curves, MXB_ERR_INVALID, "mxb_patch_create: an ENVGEN stage needs eg_levels / eg_times / eg_curves");
    // the descriptor's shape is shape 0 of mxb_patch_create2
    const mxb_envgen_shape shape = {d->eg_stages, d->eg_loop, d->eg_retrigger, d->eg_levels, d->eg_times, d->eg_curves};
    mxb_patch_desc d2 = *d;
    d2.eg_stages = 0; d2.eg_levels = d2.eg_times = d2.eg_curves = nullptr;
    return create_patch(ctx, &d2, d->eg_stages > 0 ? 1 : 0, &shape, out, "mxb_patch_create");
}

int32_t mxb_patch_create2(mxb_ctx* ctx, const mxb_patch_desc* d, int32_t n_shapes, const mxb_envgen_shape* shapes, mxb_patch** out) {
    MXB_REQUIRE(d, MXB_ERR_INVALID, "mxb_patch_create2: NULL argument");
    MXB_REQUIRE(d->eg_stages == 0, MXB_ERR_INVALID, "mxb_patch_create2: the descriptor's eg_* must be empty (eg_stages %d): the shapes come in `shapes`", d->eg_stages);
    return create_patch(ctx, d, n_shapes, shapes, out, "mxb_patch_create2");
}

int32_t mxb_patch_destroy(mxb_patch* p) {
    if (!p) return MXB_OK;
    DeviceGuard g(p->ctx->device);
    cudaDeviceSynchronize();
    delete p;
    return MXB_OK;
}

int32_t mxb_patch_set_param(mxb_patch* p, int32_t j, const double* values, int32_t mem) {
    MXB_REQUIRE(p && values, MXB_ERR_INVALID, "mxb_patch_set_param: NULL argument");
    MXB_REQUIRE(j >= 0 && j < p->n_params, MXB_ERR_INVALID, "mxb_patch_set_param: parameter %d of %d", j, p->n_params);
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_patch_set_param: mem %d", mem);
    DeviceGuard g(p->ctx->device);
    MXB_CUDA(cudaMemcpy(p->params.get() + (size_t)j * p->V, values, sizeof(double) * (size_t)p->V, mem == MXB_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice));
    return MXB_OK;
}

static int32_t patch_state_ptr(mxb_patch* p, int32_t stage, int32_t slot, double** ptr, const char* who) {
    MXB_REQUIRE(p, MXB_ERR_INVALID, "%s: NULL patch", who);
    MXB_REQUIRE(stage >= 0 && stage < p->n_stages, MXB_ERR_INVALID, "%s: stage %d of %d", who, stage, p->n_stages);
    MXB_REQUIRE(slot >= 0 && slot < patch_state_slots(p->stages[stage].op), MXB_ERR_INVALID, "%s: stage %d has %d state slots, not %d", who, stage, patch_state_slots(p->stages[stage].op), slot);
    *ptr = p->state.get() + (size_t)(p->state_base[stage] + slot) * p->V;
    return MXB_OK;
}

int32_t mxb_patch_set_state(mxb_patch* p, int32_t stage, int32_t slot, const double* values, int32_t mem) {
    double* dst = nullptr;
    int rc = patch_state_ptr(p, stage, slot, &dst, "mxb_patch_set_state");
    if (rc != MXB_OK) return rc;
    MXB_REQUIRE(values && (mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE), MXB_ERR_INVALID, "mxb_patch_set_state: bad argument");
    DeviceGuard g(p->ctx->device);
    MXB_CUDA(cudaMemcpy(dst, values, sizeof(double) * (size_t)p->V, mem == MXB_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice));
    return MXB_OK;
}

int32_t mxb_patch_get_state(mxb_patch* p, int32_t stage, int32_t slot, double* values, int32_t mem) {
    double* src = nullptr;
    int rc = patch_state_ptr(p, stage, slot, &src, "mxb_patch_get_state");
    if (rc != MXB_OK) return rc;
    MXB_REQUIRE(values && (mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE), MXB_ERR_INVALID, "mxb_patch_get_state: bad argument");
    DeviceGuard g(p->ctx->device);
    MXB_CUDA(cudaMemcpy(values, src, sizeof(double) * (size_t)p->V, mem == MXB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice));
    return MXB_OK;
}

int32_t mxb_patch_get_ring(mxb_patch* p, int32_t stage, int32_t voice, double* dst, int32_t n, int32_t mem) {
    MXB_REQUIRE(p && dst, MXB_ERR_INVALID, "mxb_patch_get_ring: NULL argument");
    MXB_REQUIRE(stage >= 0 && stage < p->n_stages && p->ring_of[stage] >= 0, MXB_ERR_INVALID, "mxb_patch_get_ring: stage %d has no delay line", stage);
    MXB_REQUIRE(voice >= 0 && voice < p->V && n >= 0 && n <= p->taps * patch_stage_rings(p->stages[stage].op), MXB_ERR_INVALID, "mxb_patch_get_ring: voice %d n %d", voice, n);
    DeviceGuard g(p->ctx->device);
    const double* src = p->rings.get() + (size_t)p->ring_of[stage] * (size_t)p->taps * (size_t)p->V + (size_t)voice;
    if (n) MXB_CUDA(cudaMemcpy2D(dst, sizeof(double), src, sizeof(double) * (size_t)p->V, sizeof(double), (size_t)n,
                                 mem == MXB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice));
    return MXB_OK;
}

int32_t mxb_patch_get_held(mxb_patch* p, int32_t m, double* values, int32_t mem) {
    double* src = nullptr;
    const int rc = patch_held_ptr(p, m, &src, "mxb_patch_get_held");
    if (rc != MXB_OK) return rc;
    MXB_REQUIRE(values && (mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE), MXB_ERR_INVALID, "mxb_patch_get_held: bad argument");
    DeviceGuard g(p->ctx->device);
    MXB_CUDA(cudaMemcpy(values, src, sizeof(double) * (size_t)p->V, mem == MXB_MEM_HOST ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice));
    return MXB_OK;
}

int32_t mxb_patch_set_held(mxb_patch* p, int32_t m, const double* values, int32_t mem) {
    double* dst = nullptr;
    const int rc = patch_held_ptr(p, m, &dst, "mxb_patch_set_held");
    if (rc != MXB_OK) return rc;
    MXB_REQUIRE(values && (mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE), MXB_ERR_INVALID, "mxb_patch_set_held: bad argument");
    DeviceGuard g(p->ctx->device);
    MXB_CUDA(cudaMemcpy(dst, values, sizeof(double) * (size_t)p->V, mem == MXB_MEM_HOST ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice));
    return MXB_OK;
}

int64_t mxb_patch_launch_count(const mxb_patch* p) { return p ? p->launches : 0; }

int32_t mxb_patch_set_mode(mxb_patch* p, int32_t mode) {
    MXB_REQUIRE(p, MXB_ERR_INVALID, "mxb_patch_set_mode: NULL patch");
    MXB_REQUIRE(mode == MXB_PATCH_INTERPRET || mode == MXB_PATCH_FUSED, MXB_ERR_INVALID, "mxb_patch_set_mode: mode %d", mode);
    if (mode == MXB_PATCH_FUSED) {          // compile now: a patch that cannot be compiled says so here, not in the audio loop
        DeviceGuard g(p->ctx->device);
        const int rc = patch_fused_load(p);
        if (rc != MXB_OK) return rc;
    }
    p->mode = mode;
    return MXB_OK;
}

int32_t mxb_patch_get_mode(const mxb_patch* p) { return p ? p->mode : MXB_ERR_INVALID; }

int32_t mxb_patch_codegen(const mxb_patch_desc* d, char* buf, int64_t cap, int64_t* needed, int32_t compile) {
    MXB_REQUIRE(d && d->stages && needed, MXB_ERR_INVALID, "mxb_patch_codegen: NULL argument");
    const int rc = validate_stages(d, kMaxEgShapes, "mxb_patch_codegen");      // the shapes are kernel arguments: any of them may be set
    if (rc != MXB_OK) return rc;
    const std::string src = patch_generate_source(d->stages, d->n_stages, d->n_params, d->consts, d->n_consts, d->n_inputs, d->input_types);
    *needed = (int64_t)src.size() + 1;
    if (buf && cap > 0) { const size_t n = src.size() + 1 <= (size_t)cap ? src.size() : (size_t)cap - 1; memcpy(buf, src.data(), n); buf[n] = 0; }
    if (compile) {
        std::vector<char> cubin;
        const int crc = patch_compile(src, cubin);
        if (crc != MXB_OK) return crc;
        MXB_REQUIRE(!cubin.empty(), MXB_ERR_STATE, "mxb_patch_codegen: the compiler returned no code");
    }
    return MXB_OK;
}

int32_t mxb_patch_process(mxb_patch* p, int32_t n_frames, const void* const* inputs, double* out, double* mix, int32_t mem, void* stream_) {
    NvtxRange nvtx_("mxb_patch_process");
    MXB_REQUIRE(p, MXB_ERR_INVALID, "mxb_patch_process: NULL patch");
    MXB_REQUIRE(n_frames >= 0 && n_frames <= p->max_frames, MXB_ERR_INVALID, "mxb_patch_process: n_frames %d (max_frames %d)", n_frames, p->max_frames);
    MXB_REQUIRE(mem == MXB_MEM_HOST || mem == MXB_MEM_DEVICE, MXB_ERR_INVALID, "mxb_patch_process: mem %d", mem);
    MXB_REQUIRE(p->n_inputs == 0 || inputs, MXB_ERR_INVALID, "mxb_patch_process: the patch reads %d input streams, inputs is NULL", p->n_inputs);
    for (int i = 0; i < p->n_inputs; ++i) {
        MXB_REQUIRE(inputs[i], MXB_ERR_INVALID, "mxb_patch_process: input stream %d is NULL", i);
        if (p->in_type[i] == MXB_IN_EVENTS) {
            const int rc = check_events(p, i, (const mxb_events*)inputs[i], mem == MXB_MEM_HOST);
            if (rc != MXB_OK) return rc;
        }
    }
    if (mix) {     // before any kernel runs: a refused call leaves every stage's state untouched
        const int rc = mix_bus_admit(p->ex, n_frames, "mxb_patch_process");
        if (rc != MXB_OK) return rc;
    }
    if (n_frames == 0) return MXB_OK;
    DeviceGuard g(p->ctx->device);
    cudaStream_t s = (cudaStream_t)stream_;
    const size_t V = (size_t)p->V, nb = sizeof(double) * (size_t)n_frames * V;
    PatchArgs a;
    memset(&a, 0, sizeof(a));
    const bool host = mem == MXB_MEM_HOST;
    for (int i = 0; i < p->n_inputs; ++i) {
        a.in_kind[i] = (unsigned char)p->in_type[i];
        if (p->in_type[i] == MXB_IN_EVENTS) {
            const int rc = stage_events(p, i, (const mxb_events*)inputs[i], host, s, &a.ev[p->ev_of[i]]);
            if (rc != MXB_OK) return rc;
            a.ev_of[i] = p->ev_of[i];
            continue;
        }
        const unsigned char* d_in;
        const int rc = stage_in(host, (const unsigned char*)inputs[i], patch_input_bytes(p->in_type[i], (size_t)n_frames, V), p->in_stage[i], s, &d_in);
        if (rc != MXB_OK) return rc;
        a.inputs[i] = d_in;
    }
    double *d_out, *d_mix;
    int rc = stage_out(host, out, (size_t)n_frames * V, p->out_stage, s, &d_out);
    if (rc == MXB_OK) rc = stage_out(host, mix, (size_t)n_frames * 2, p->mix_dev, s, &d_mix);
    if (rc != MXB_OK) return rc;
    const int grid = (int)((V + kPatchThreads - 1) / kPatchThreads);
    const int W = grid * (kPatchThreads / 32);
    if (mix) { rc = p->partials.grow((size_t)p->max_frames * 2 * (size_t)W, s); if (rc != MXB_OK) return rc; }
    a.V = p->V; a.n_frames = n_frames; a.n_stages = p->n_stages; a.n_params = p->n_params; a.n_state = p->n_state; a.W = W; a.taps = p->taps;
    a.sr = (double)(size_t)p->ctx->sample_rate;
    a.stages = p->d_stages.get(); a.state_base = p->d_state_base.get(); a.ring_of = p->d_ring_of.get(); a.consts = p->d_consts.get();
    a.params = p->params.get(); a.state = p->state.get(); a.out = d_out; a.partials = mix ? p->partials.get() : nullptr; a.rings = p->rings.get();
    const double* sine = p->ctx->d_sine.get();
    a.sine = sine; a.transition = sine ? sine + 514 : nullptr; a.sine_before = p->ctx->sine_before;
    memcpy(a.eg_n, p->eg_n, sizeof(a.eg_n)); memcpy(a.eg_loop, p->eg_loop, sizeof(a.eg_loop)); memcpy(a.eg_retrigger, p->eg_retrigger, sizeof(a.eg_retrigger));
    memcpy(a.eg, p->eg, sizeof(a.eg));
    a.n_ev = p->n_ev; a.held = p->held.get();
    if (p->mode == MXB_PATCH_FUSED) {
        // the kernel generated for this stage list (patch_fuse.cu): compiled on first use, then launched like any other
        rc = patch_fused_load(p);
        if (rc == MXB_OK) rc = patch_fused_launch(p, a, grid, s);
        if (rc != MXB_OK) return rc;
    } else {
        const size_t smem = sizeof(double) * (size_t)(kMaxRegs + p->n_params + p->n_state + 3 * p->n_ev) * kPatchThreads;
        void (*kernel)(const PatchArgs) = p->n_ev ? (p->n_shapes > 1 ? patch_kernel<true, true> : patch_kernel<false, true>)
                                                  : (p->n_shapes > 1 ? patch_kernel<true, false> : patch_kernel<false, false>);
        rc = smem_limit_at_least((const void*)kernel, smem, "patch_kernel");
        if (rc != MXB_OK) return rc;
        kernel<<<grid, kPatchThreads, smem, s>>>(a);
        MXB_CUDA(cudaGetLastError());
    }
    p->launches += 1;
    if (mix) {
        rc = mix_bus_reduce(p->ex, p->partials.get(), W, n_frames, d_mix, s);
        if (rc != MXB_OK) return rc;
        p->launches += 1;
    }
    if (host) {
        if (out) MXB_CUDA(cudaMemcpyAsync(out, d_out, nb, cudaMemcpyDeviceToHost, s));
        if (mix) MXB_CUDA(cudaMemcpyAsync(mix, d_mix, sizeof(double) * (size_t)n_frames * 2, cudaMemcpyDeviceToHost, s));
        MXB_CUDA(cudaStreamSynchronize(s));
        if (mix) return mix_bus_status(p->ex, "mxb_patch_process");      // the call is synchronous in this mode: a timed-out exchange is an error of THIS call
    }
    return MXB_OK;
}

int32_t mxb_patch_set_exchange(mxb_patch* p, mxb_exchange* ex) {
    MXB_REQUIRE(p, MXB_ERR_INVALID, "mxb_patch_set_exchange: NULL patch");
    const int rc = mix_bus_attach(ex, p->ctx->device, "mxb_patch_set_exchange");
    if (rc != MXB_OK) return rc;
    p->ex = ex;
    return MXB_OK;
}

}  // extern "C"
