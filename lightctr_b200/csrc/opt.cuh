// lightctr_b200/csrc/opt.cuh -- per-coordinate updater arithmetic shared by every applier: the sparse apply kernel
// (opt.cu), the compact updater (fm_fused.cuh), the feature-major backwards (fm.cu, csc.cu, ffm_grouped.cu) and the
// owner-side merge of several GPUs (dist.cu).
//
// Contract: a coordinate whose batch gradient is exactly zero keeps its parameter and its state, under all nine rules.
// An applier may therefore visit any set of coordinates that holds the nonzero ones -- whole rows of the batch's
// features, only their nonzero 4-wide slices, or only the rows a merge saw a nonzero record for -- and every applier
// gives the same result.  tests/test_updaters_gpu.py holds each applier to the oracle bit for bit under every rule.
#pragma once
#include <math.h>

#include <type_traits>

#include "common.cuh"

namespace lctr {

struct OptParams {
    int opt;
    float invB;       // (float)(1.0 / minibatch)  (Adagrad: avx_vecScale(grad, grad, len, 1.0/B))
    float mb;         // (float)minibatch          (Adam: grad / minibatch)
    float lr;
    float beta1;
    float corrW, corrV;  // Adam bias corrections of the W call and the V call (iter++ per call)
    float alpha, beta, l1, l2;
    float ema;        // RMSprop: GradientUpdater::__global_ema_rate
    int tensor_v;     // LCTR_OPT_PS_SGD: the V call uses the tensor SGD form (Wide&Deep tensors, paramserver.h:232-237)
};

// updaters that carry a second state array (FTRL n, Adam v)
__host__ __device__ __forceinline__ bool opt_two_states(int opt) {
    return opt == LCTR_OPT_FTRL || opt == LCTR_OPT_ADAM || opt == LCTR_OPT_ADADELTA || opt == LCTR_OPT_PS_DCASGD || opt == LCTR_OPT_PS_DCASGDA;
}

// one coordinate; arithmetic order as in the reference (compiled with -fmad=false)
__device__ __forceinline__ void update_one(const OptParams& P, float corr, float& w, float g, float& s1, float& s2) {
    if (P.opt == LCTR_OPT_ADAGRAD) {
        const float g1 = g * P.invB;
        if (g1 != 0.f) {
            s1 = s1 + g1 * g1;
            w = (float)((double)w - (double)(P.lr * g1) / sqrt((double)s1 + 1e-7));
        }
    } else if (P.opt == LCTR_OPT_FTRL) {
        if (g != 0.f) {
            const float g2 = g * g;
            const float sigma = (sqrtf(s2 + g2) - sqrtf(s2)) / P.alpha;
            s1 = s1 + (g - sigma * w);  // z
            s2 = s2 + g2;               // n
            if (fabsf(s1) <= P.l1) {
                w = 0.f;
            } else {
                float t = s1;
                if (t >= 0.f) t -= P.l1; else t += P.l1;
                w = -t / ((P.beta + sqrtf(s2)) / P.alpha + P.l2);
            }
        }
    } else if (P.opt == LCTR_OPT_RMSPROP) {  // RMSpropUpdater_Num::update, gradientUpdater.h:216-229
        float g1 = g / P.mb;
        if (g1 != 0.f) {
            s1 = (float)((double)(s1 * P.ema) + (1.0 - (double)P.ema) * (double)g1 * (double)g1);
            const float tmp = (float)(1.0 / ((double)s1 + 1e-7));
            g1 = g1 * sqrtf(tmp);
            w = w - P.lr * g1;
        }
    } else if (P.opt == LCTR_OPT_ADADELTA) {  // AdadeltaUpdater_Num::update, momentumUpdater.h:91-106 (s1 = E[g^2], s2 = E[d^2])
        float g1 = g / P.mb;
        if (g1 != 0.f) {
            s1 = (float)((double)(s1 * P.beta1) + (1.0 - (double)P.beta1) * (double)g1 * (double)g1);
            const float tmp = (float)(((double)s2 + 1e-7) / ((double)s1 + 1e-7));
            g1 = g1 * sqrtf(tmp);
            s2 = (float)((double)(s2 * P.beta1) + (1.0 - (double)P.beta1) * (double)g1 * (double)g1);
            w = w - g1;
        }
    } else if (P.opt >= LCTR_OPT_PS_SGD) {
        // ParamServer push handler (distribut/paramserver.h:232-300).  The reference's Value operators MUTATE their left
        // operand (distributed_algo_abst.h:39-72: `a * b` is `a.w *= b.w; return a`), which the sequences below follow.
        // corr == 0: scalar parameters (the W call); corr != 0: tensors (the V call) -- Wide&Deep tensors take the tensor
        // SGD form under LCTR_OPT_PS_SGD when P.tensor_v is set.
        // A zero gradient is never pushed (Value::checkPreferredValue, push.h:62-65), so it changes nothing here either:
        // without this, DCASGD would still copy w into its shadow and DCASGDA would still decay its accumulator.
        if (g == 0.f) return;
        if (P.opt == LCTR_OPT_PS_SGD) {
            if (corr != 0.f && P.tensor_v) {  // :232-237  scaler = -lr / minibatch (double expression narrowed to float)
                const float scaler = (float)(-1.0 * (double)P.lr / (double)P.mb);
                w = w + g * scaler;
            } else {                          // :295-300  data - grad / ((float)minibatch / lr)
                w = w - g / (P.mb / P.lr);
            }
        } else if (P.opt == LCTR_OPT_PS_ADAGRAD) {  // :288-294 (s1 = data_accum, initialised to 1e-7 :323)
            // `TValue grad = data_pair.second / minibatch` divides the PUSHED value in place (Value::operator/ mutates and
            // returns *this, distributed_algo_abst.h:56-63), so the step below uses g / minibatch, not g -- pinned by the
            // reference cluster's Adagrad curve (tests/golden/wnd_ref_curve.json)
            const float gm = g / P.mb;
            float grad = gm * gm;
            s1 = s1 + grad;
            float sq = (float)sqrt((double)s1 + 1e-7);
            sq = sq / P.lr;
            w = w - gm / sq;
        } else if (P.opt == LCTR_OPT_PS_DCASGD) {   // :252-267 (s2 = shadow copy of worker 0)
            float grad = g / P.mb;
            float reserve = grad;
            grad = grad * grad;
            const float cur = w - s2;
            grad = grad * cur;
            grad = grad * 0.1f;
            reserve = reserve + grad;
            reserve = reserve * P.lr;
            w = w - reserve;
            s2 = w;
        } else {                                    // DCASGDA :268-286 (s1 = data_accum, s2 = shadow copy)
            float grad = g / P.mb;
            s1 = s1 * 0.95f;
            grad = grad * grad;
            grad = grad * (1 - 0.95f);
            s1 = s1 + grad;
            float reserve = grad;  // the reference copies `grad` AFTER it was overwritten by 0.05 g^2 (:277)
            const float sq = (float)sqrt((double)s1 + 1e-7);
            grad = grad * grad;
            const float cur = w - s2;
            grad = grad * cur;
            grad = grad * 0.1f;
            grad = grad / sq;
            reserve = reserve + grad;
            reserve = reserve * P.lr;
            w = w - reserve;
            s2 = w;
        }
    } else {  // Adam (both moments decay with beta1 -- reference quirk, momentumUpdater.h:197-201)
        const float g1 = g / P.mb;
        if (g1 != 0.f) {
            s1 = (float)((double)(s1 * P.beta1) + (1.0 - (double)P.beta1) * (double)g1);
            s2 = (float)((double)(s2 * P.beta1) + (1.0 - (double)P.beta1) * (double)g1 * (double)g1);
            const float tmp = (float)((double)s1 / ((double)sqrtf(s2) + 1e-7));
            w = w - P.lr * corr * tmp;
        }
    }
}


// host: snapshot of the hyper-parameters for one step (advances the Adam call counter)
// pick(std::integral_constant<int, OPT>()) for the updater opt: the instance of a kernel specialised per optimizer
template <typename Pick>
auto by_opt(int opt, Pick&& pick) {
    return by_value<LCTR_OPT_ADAGRAD, LCTR_OPT_FTRL, LCTR_OPT_ADAM, LCTR_OPT_RMSPROP, LCTR_OPT_ADADELTA, LCTR_OPT_PS_SGD,
                    LCTR_OPT_PS_ADAGRAD, LCTR_OPT_PS_DCASGD, LCTR_OPT_PS_DCASGDA>(opt, pick);
}

inline OptParams make_opt_params(lctr_ctx* c, int64_t rows_in_step) {
    const lctr_cfg& cf = c->cfg;
    OptParams P;
    P.opt = cf.optimizer;
    const uint64_t mb = cf.minibatch_size ? cf.minibatch_size : (uint64_t)rows_in_step;
    P.invB = (float)(1.0 / (double)mb);
    P.mb = (float)mb;
    P.lr = cf.learning_rate;
    P.beta1 = cf.momentum;
    P.corrW = P.corrV = 1.f;
    if (cf.optimizer == LCTR_OPT_ADAM) {
        // iter++ per update() call: W first, then V (train_fm_algo.cpp:120-126 order)
        size_t it = ++c->adam_iter;
        P.corrW = (float)(sqrt(1 - pow((double)cf.momentum_adam2, (double)it)) / (1 - pow((double)cf.momentum, (double)it)));
        it = ++c->adam_iter;
        P.corrV = (float)(sqrt(1 - pow((double)cf.momentum_adam2, (double)it)) / (1 - pow((double)cf.momentum, (double)it)));
    }
    P.ema = cf.ema_rate != 0.f ? cf.ema_rate : 0.99f;
    P.tensor_v = cf.model == LCTR_MODEL_WND ? 1 : 0;
    if (cf.optimizer >= LCTR_OPT_PS_SGD) { P.corrW = 0.f; P.corrV = 1.f; }  // W call / V call marker for the PS rules
    P.alpha = cf.ftrl_alpha; P.beta = cf.ftrl_beta; P.l1 = cf.ftrl_lambda1; P.l2 = cf.ftrl_lambda2;
    return P;
}

}  // namespace lctr
