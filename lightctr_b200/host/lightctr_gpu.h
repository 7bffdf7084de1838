// lightctr_b200/host/lightctr_gpu.h -- C++ host shims with the reference's trainer class surface.
//
// Drop-in for the FM / FFM / NFM hot path of cnkuangshi/LightCTR: same class names, constructor
// signatures, public members and call sequence as
//     FM_Algo_Abst        LightCTR/fm_algo_abst.h:37-172
//     Train_FM_Algo       LightCTR/train/train_fm_algo.h:21-58
//     Train_FFM_Algo      LightCTR/train/train_ffm_algo.h:22-66
//     Train_NFM_Algo      LightCTR/train/train_nfm_algo.h:18-77
//     FM_Predict          LightCTR/predict/fm_predict.h:17-39
//     Layer_Base / Fully_Conn_Layer / DL_Algo_Abst   LightCTR/train/layer/layer_abst.h:25-83, fullyconnLayer.h:15-238,
//                         dl_algo_abst.h:25-246 (minibatch-batched: see the comment above Layer_Base below)
//     Distributed_Algo_Abst   LightCTR/distributed_algo_abst.h:86-292 (one process per GPU instead of ZeroMQ workers)
//     GradientUpdater / MomentumUpdater statics   LightCTR/util/gradientUpdater.h:36-42, main.cpp:64-73
// but every Train()/Predict() lowers to the C ABI of include/lightctr_b200.h (CUDA, sm_90a).  A caller
// such as the reference's main.cpp:144-162,228-253 compiles unchanged against this header inside
// `namespace lightctr_b200` (see INTEGRATION.md).  Error behaviour follows the reference: print + exit(1)
// (fm_algo_abst.h:79-82).  Host-side randomness uses libc rand() in the reference's call order
// (util/random.h:21-58,82), so srand(seed) reproduces its initialisation bit for bit.
#ifndef LIGHTCTR_GPU_H
#define LIGHTCTR_GPU_H

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include <algorithm>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/lightctr_b200.h"

namespace lightctr_b200 {

// ---- util/gradientUpdater.h:36-42, util/momentumUpdater.h: process-global hyper-parameters ----------------
struct GradientUpdater {
    static size_t __global_minibatch_size;
    static float __global_learning_rate;
    static float __global_ema_rate;
    static float __global_sparse_rate;
    static float __global_lambdaL2, __global_lambdaL1;
    static bool __global_bTraining;
};
struct MomentumUpdater {
    static float __global_momentum;
    static float __global_momentum_adam2;
};
// Define once in the application (the reference does the same in main.cpp:64-73):
#define LIGHTCTR_B200_DEFINE_GLOBALS                                                   \
    size_t lightctr_b200::GradientUpdater::__global_minibatch_size(50);                \
    float lightctr_b200::GradientUpdater::__global_learning_rate(0.05);                \
    float lightctr_b200::GradientUpdater::__global_ema_rate(0.99);                     \
    float lightctr_b200::GradientUpdater::__global_sparse_rate(0.8);                   \
    float lightctr_b200::GradientUpdater::__global_lambdaL2(0.001f);                   \
    float lightctr_b200::GradientUpdater::__global_lambdaL1(1e-5);                     \
    float lightctr_b200::MomentumUpdater::__global_momentum(0.8);                      \
    float lightctr_b200::MomentumUpdater::__global_momentum_adam2(0.999);              \
    bool lightctr_b200::GradientUpdater::__global_bTraining(true);

// ---- util/random.h:21-58,82 ------------------------------------------------------------------------------
inline double UniformNumRand() { return static_cast<double>(rand()) / (static_cast<double>(RAND_MAX) + 1.0); }
inline double UniformNumRand2() { return (static_cast<double>(rand()) + 1.0) / (static_cast<double>(RAND_MAX) + 2.0); }
inline double GaussRand() {
    static double V1, V2, S;
    static int phase = 0;
    double X;
    if (phase == 0) {
        do {
            V1 = 2.0 * UniformNumRand2() - 1.0;
            V2 = 2.0 * UniformNumRand2() - 1.0;
            S = V1 * V1 + V2 * V2;
        } while (S >= 1.0 || S == 0.0);
        X = V1 * sqrt(-2.0 * log(S) / S);
    } else {
        X = V2 * sqrt(-2.0 * log(S) / S);
    }
    phase = 1 - phase;
    return X;
}
inline bool SampleBinary(double p) { return UniformNumRand() < p; }

inline void lctr_die(const char* what) {
    std::cout << what << ": " << lctr_last_error() << std::endl;
    exit(1);
}
#define LCTR_OK(call) do { if ((call) != 0) ::lightctr_b200::lctr_die(#call); } while (0)

struct FMFeature {  // fm_algo_abst.h:29-35
    size_t first;   // feature id
    float second;   // value
    size_t field;
    FMFeature(size_t _first, float _second, size_t _field) : first(_first), second(_second), field(_field) {}
};

class FM_Algo_Abst {
public:
    FM_Algo_Abst(std::string _dataPath, size_t _factor_cnt, size_t _field_cnt = 0, size_t _feature_cnt = 0)
        : feature_cnt(_feature_cnt), field_cnt(_field_cnt), factor_cnt(_factor_cnt) {
        proc_cnt = 1;  // kept for source compatibility (fm_algo_abst.h:42); parallelism lives on the device
        loadDataRow(_dataPath);
        init();
    }
    virtual ~FM_Algo_Abst() {
        delete[] W;
        delete[] V;
        delete[] sumVX;
        if (ds) lctr_free_dataset(ds);
        if (ctx) lctr_destroy(ctx);
    }
    void init() {  // fm_algo_abst.h:53-68
        W = new float[feature_cnt];
        memset(W, 0, sizeof(float) * feature_cnt);
        size_t memsize = feature_cnt * factor_cnt;
        if (field_cnt > 0) memsize = feature_cnt * field_cnt * factor_cnt;
        V = new float[memsize];
        const float scale = 1.0 / sqrt(factor_cnt);
        for (size_t i = 0; i < memsize; i++) V[i] = GaussRand() * scale;
        sumVX = NULL;
    }
    void loadDataRow(std::string dataPath) {  // fm_algo_abst.h:70-107 (parser lives in the library, bit-exact)
        if (lctr_load_libffm(dataPath.c_str(), field_cnt, feature_cnt, &ds) != 0) {
            std::cout << "open file error!" << std::endl;
            exit(1);
        }
        feature_cnt = ds->feature_cnt;
        field_cnt = ds->field_cnt;
        dataRow_cnt = (size_t)ds->rows;
        dataSet.clear();  // the AoS view the reference exposes publicly (fm_algo_abst.h:156)
        dataSet.resize(dataRow_cnt);
        for (size_t r = 0; r < dataRow_cnt; r++)
            for (int64_t e = ds->row_ptr[r]; e < ds->row_ptr[r + 1]; e++)
                dataSet[r].emplace_back(FMFeature(ds->fid[e], ds->val[e], ds->field[e]));
        label.assign(ds->label, ds->label + ds->label_cnt);
    }
    void saveModel(size_t epoch) {  // fm_algo_abst.h:109-135
        char buffer[1024];
        snprintf(buffer, 1024, "%d", (int)epoch);
        std::string filename = buffer;
        std::ofstream md("./output/model_epoch_" + filename + ".txt");
        if (!md.is_open()) {
            std::cout << "save model open file error" << std::endl;
            exit(1);
        }
        for (size_t fid = 0; fid < feature_cnt; fid++)
            if (W[fid] != 0) md << fid << ":" << W[fid] << " ";
        md << std::endl;
        for (size_t fid = 0; fid < feature_cnt; fid++) {
            md << fid << ":";
            for (size_t f = 0; f < factor_cnt; f++) md << *getV(fid, f) << " ";
            md << std::endl;
        }
        md.close();
    }
    virtual void Train() = 0;

    float L2Reg_ratio;
    float* W;
    size_t feature_cnt, proc_cnt, field_cnt, factor_cnt;
    size_t dataRow_cnt;
    float *V, *sumVX;
    inline float* getV(size_t fid, size_t facid) const { return &V[fid * factor_cnt + facid]; }
    inline float* getV_field(size_t fid, size_t fieldid, size_t facid) const {
        return &V[fid * field_cnt * factor_cnt + fieldid * factor_cnt + facid];
    }
    inline float* getSumVX(size_t rid, size_t facid) const { return &sumVX[rid * factor_cnt + facid]; }
    std::vector<std::vector<FMFeature> > dataSet;
    std::vector<int> label;

    // ---- device side ---------------------------------------------------------------------------------------
    lctr_ctx* ctx = nullptr;
    lctr_dataset* ds = nullptr;
    int updater = LCTR_OPT_ADAGRAD;  // the reference's `AdagradUpdater_Num updater;` member (fm_algo_abst.h:166)
    int deterministic = 1;           // ascending-row accumulation (== the reference's canonical proc_cnt=1 order)
    int mlp_precision = LCTR_MLP_FP32;  // NFM dense layers: reference-order fp32 (parity) or LCTR_MLP_BF16 (tensor cores)

protected:
    float __loss;
    float __accuracy;
    void make_ctx(int model, size_t minibatch, size_t csc_block, int n_hidden = 0, const uint32_t* hidden = nullptr) {
        lctr_cfg cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.abi_version = LCTR_ABI_VERSION;
        cfg.model = model;
        cfg.optimizer = updater;
        cfg.feature_cnt = feature_cnt;
        cfg.field_cnt = model == LCTR_MODEL_FFM ? (uint32_t)field_cnt : 0;
        cfg.factor_cnt = (uint32_t)factor_cnt;
        cfg.learning_rate = GradientUpdater::__global_learning_rate;
        cfg.l2_reg = L2Reg_ratio;
        cfg.minibatch_size = minibatch;
        cfg.momentum = MomentumUpdater::__global_momentum;
        cfg.momentum_adam2 = MomentumUpdater::__global_momentum_adam2;
        cfg.ema_rate = GradientUpdater::__global_ema_rate;  // RMSpropUpdater_Num (updater = LCTR_OPT_RMSPROP)
        cfg.n_hidden = n_hidden;
        for (int i = 0; i < n_hidden; i++) cfg.hidden[i] = hidden[i];
        cfg.activation = LCTR_ACT_SIGMOID;
        cfg.mlp_precision = mlp_precision;
        cfg.deterministic = deterministic;
        cfg.csc_row_block = csc_block;
        LCTR_OK(lctr_create(&cfg, &ctx));
        LCTR_OK(lctr_upload_params(ctx, W, V));
        bool ones = true;
        for (int64_t e = 0; e < ds->nnz && ones; e++) ones = ds->val[e] == 1.0f;
        LCTR_OK(lctr_upload_batch(ctx, 0, ds->rows, ds->nnz, ds->row_ptr, ds->fid, ds->field, ones ? nullptr : ds->val,
                                  ds->label));
        LCTR_OK(lctr_sync(ctx));
    }
};

class Train_FM_Algo : public FM_Algo_Abst {
public:
    Train_FM_Algo(std::string _dataPath, size_t _epoch_cnt, size_t _factor_cnt)
        : FM_Algo_Abst(_dataPath, _factor_cnt), epoch_cnt(_epoch_cnt) {
        if (feature_cnt == 0) { std::cout << "assert(feature_cnt != 0)" << std::endl; exit(1); }
        L2Reg_ratio = 0.001f;  // train_fm_algo.cpp:13
        sumVX = new float[dataRow_cnt * factor_cnt];
        memset(sumVX, 0, sizeof(float) * dataRow_cnt * factor_cnt);
    }
    void Train() {  // train_fm_algo.cpp:35-61
        GradientUpdater::__global_bTraining = true;
        GradientUpdater::__global_minibatch_size = dataRow_cnt;
        if (!ctx) make_ctx(LCTR_MODEL_FM, 0, 0);
        for (size_t i = 0; i < epoch_cnt; i++) {
            LCTR_OK(lctr_train_step(ctx, 0, 0, (int64_t)dataRow_cnt, &__loss, &__accuracy));
            printf("Epoch %zu Train Loss = %f Accuracy = %f\n", i, __loss, __accuracy / dataRow_cnt);
        }
        LCTR_OK(lctr_download_params(ctx, W, V));  // FM_Predict / saveModel read these (fm_predict.cpp:25-32)
        LCTR_OK(lctr_download_sumvx(ctx, 0, sumVX));
        GradientUpdater::__global_bTraining = false;
    }
    float last_loss() const { return __loss; }

private:
    size_t epoch_cnt;
};

class Train_FFM_Algo : public FM_Algo_Abst {
public:
    Train_FFM_Algo(std::string _dataPath, size_t _epoch_cnt, size_t _factor_cnt, size_t _field_cnt)
        : FM_Algo_Abst(_dataPath, _factor_cnt, _field_cnt), epoch(_epoch_cnt) {
        L2Reg_ratio = 0.001f;
        printf("Training FFM\n");
    }
    void Train() {  // train_ffm_algo.cpp:23-49
        GradientUpdater::__global_bTraining = true;
        GradientUpdater::__global_minibatch_size = dataRow_cnt;
        if (!ctx) make_ctx(LCTR_MODEL_FFM, 0, 0);
        for (size_t i = 0; i < epoch; i++) {
            LCTR_OK(lctr_train_step(ctx, 0, 0, (int64_t)dataRow_cnt, &__loss, &__accuracy));
            printf("Epoch %zu Train Loss = %f Accuracy = %f\n", i, __loss, __accuracy / dataRow_cnt);
        }
        LCTR_OK(lctr_download_params(ctx, W, V));
        GradientUpdater::__global_bTraining = false;
    }
    float last_loss() const { return __loss; }

private:
    size_t epoch;
};

// Host shadow of Fully_Conn_Layer (train/layer/fullyconnLayer.h:36-61,194-206): initial values and the dropout
// mask come from the reference's rand() stream in the reference's order; the arithmetic runs on the device.
struct Fully_Conn_Layer_Host {
    size_t in, out;
    std::vector<float> weight, bias, mask;
    Fully_Conn_Layer_Host(size_t _in, size_t _out) : in(_in), out(_out), weight(_in * _out), bias(_out, 0.f), mask(_out) {
        for (size_t i = 0; i < out; i++) {
            mask[i] = SampleBinary(GradientUpdater::__global_sparse_rate) ? 1. : 0.;
            for (size_t j = 0; j < in; j++) weight[i * in + j] = UniformNumRand() - 0.5f;
        }
    }
    void resample() {
        for (size_t i = 0; i < out; i++) mask[i] = SampleBinary(GradientUpdater::__global_sparse_rate) ? 1. : 0.;
    }
};

class Train_NFM_Algo : public FM_Algo_Abst {
public:
    Train_NFM_Algo(std::string _dataPath, size_t _epoch_cnt, size_t _factor_cnt, size_t _hidden_layer_size)
        : FM_Algo_Abst(_dataPath, _factor_cnt), epoch(_epoch_cnt), hidden_layer_size(_hidden_layer_size) {
        L2Reg_ratio = 0.001f;
        batch_size = GradientUpdater::__global_minibatch_size;  // train_nfm_algo.cpp:13
        sumVX = new float[dataRow_cnt * factor_cnt];
        memset(sumVX, 0, sizeof(float) * dataRow_cnt * factor_cnt);
        layers.emplace_back(factor_cnt, hidden_layer_size);  // :21-27
        layers.emplace_back(hidden_layer_size, 1);
        hidden_sizes.push_back((uint32_t)hidden_layer_size);
    }
    // config C4: the Fully_Conn_Layer chain factor_cnt -> hidden[0] -> ... -> 1 (Layer_Base's prevLayer / nextLayer
    // chaining, layer_abst.h:27-40); RNG order = construction order, input to output, like the reference's ctor
    Train_NFM_Algo(std::string _dataPath, size_t _epoch_cnt, size_t _factor_cnt, const std::vector<size_t>& _hidden)
        : FM_Algo_Abst(_dataPath, _factor_cnt), epoch(_epoch_cnt), hidden_layer_size(_hidden.empty() ? 0 : _hidden[0]) {
        if (_hidden.empty() || _hidden.size() > LCTR_MAX_LAYERS) { std::cout << "NFM needs 1.." << LCTR_MAX_LAYERS << " hidden layers" << std::endl; exit(1); }
        L2Reg_ratio = 0.001f;
        batch_size = GradientUpdater::__global_minibatch_size;
        sumVX = new float[dataRow_cnt * factor_cnt];
        memset(sumVX, 0, sizeof(float) * dataRow_cnt * factor_cnt);
        size_t in = factor_cnt;
        for (size_t h : _hidden) { layers.emplace_back(in, h); hidden_sizes.push_back((uint32_t)h); in = h; }
        layers.emplace_back(in, 1);
    }
    void Train() {  // train_nfm_algo.cpp:30-54
        GradientUpdater::__global_bTraining = true;
        if (!ctx) {
            make_ctx(LCTR_MODEL_NFM, GradientUpdater::__global_minibatch_size, batch_size, (int)hidden_sizes.size(),
                     hidden_sizes.data());
            for (size_t l = 0; l < layers.size(); l++) {
                LCTR_OK(lctr_mlp_upload(ctx, (int)l, layers[l].weight.data(), layers[l].bias.data()));
                LCTR_OK(lctr_mlp_set_mask(ctx, (int)l, layers[l].mask.data()));
            }
        }
        for (size_t i = 0; i < epoch; i++) {
            loss = 0;
            accuracy = 0;
            const size_t minibatch_epoch = (dataRow_cnt + batch_size - 1) / batch_size;
            for (size_t p = 0; p < minibatch_epoch; p++) {
                const size_t start_pos = p * batch_size;
                float l = 0, c = 0;
                LCTR_OK(lctr_train_step(ctx, 0, (int64_t)start_pos, (int64_t)std::min(start_pos + batch_size, dataRow_cnt), &l, &c));
                loss += l;
                accuracy += (size_t)c;
                for (size_t li = 0; li < layers.size(); li++) {  // applyBatchGradient re-draws the masks
                    layers[li].resample();
                    LCTR_OK(lctr_mlp_set_mask(ctx, (int)li, layers[li].mask.data()));
                }
            }
            printf("Epoch %zu loss = %f accuracy = %f\n", i, loss, 1.0 * accuracy / dataRow_cnt);
        }
        LCTR_OK(lctr_download_params(ctx, W, V));
        LCTR_OK(lctr_download_sumvx(ctx, 0, sumVX));
        for (size_t l = 0; l < layers.size(); l++)
            LCTR_OK(lctr_mlp_download(ctx, (int)l, layers[l].weight.data(), layers[l].bias.data()));
        GradientUpdater::__global_bTraining = false;
    }
    float last_loss() const { return loss; }
    std::vector<Fully_Conn_Layer_Host> layers;
    std::vector<uint32_t> hidden_sizes;

private:
    size_t epoch, batch_size, hidden_layer_size;
    float loss;
    size_t accuracy;
};

// predict/fm_predict.{h,cpp}.  The reference's loader drops the first feature of every test row and every fid
// >= the training feature_cnt (:117-126); its FM branch adds 0.5*|sumVX_train[rid]|^2 of the TRAINING row with the
// same index (:27-32).  Both quirks are reproduced (quirks = false gives the mathematically intended predictor).
class FM_Predict {
public:
    FM_Predict(FM_Algo_Abst* p, std::string _testDataPath, bool with_valid_label, bool quirks = true)
        : fm(p), quirks_(quirks) {
        (void)with_valid_label;
        lctr_dataset* t = nullptr;
        if (lctr_load_libffm(_testDataPath.c_str(), 0, 0, &t) != 0) {
            std::cout << "open file error!" << std::endl;
            exit(1);
        }
        row_ptr.push_back(0);
        for (int64_t r = 0; r < t->rows; r++) {
            const size_t before = fid.size();
            for (int64_t e = t->row_ptr[r] + (quirks ? 1 : 0); e < t->row_ptr[r + 1]; e++) {
                if (t->fid[e] < fm->feature_cnt) {
                    fid.push_back(t->fid[e]); field.push_back(t->field[e]); val.push_back(t->val[e]);
                }
            }
            if (fid.size() == before) continue;
            row_ptr.push_back((int64_t)fid.size());
            test_label.push_back(t->label[quirks ? (int64_t)test_label.size() : r]);
        }
        test_dataRow_cnt = row_ptr.size() - 1;
        lctr_free_dataset(t);
    }
    void Predict(std::string savePath) {  // fm_predict.cpp:12-90
        ans.resize(test_dataRow_cnt);
        LCTR_OK(lctr_upload_batch(fm->ctx, 1, (int64_t)test_dataRow_cnt, (int64_t)fid.size(), row_ptr.data(), fid.data(),
                                  field.data(), val.data(), test_label.data()));
        const bool is_ffm = fm->sumVX == NULL;
        LCTR_OK(lctr_predict(fm->ctx, 1, (quirks_ && !is_ffm) ? 0 : -1, ans.data()));
        float loss = 0;
        int correct = 0;
        for (size_t i = 0; i < test_label.size(); i++) {
            loss += (int)test_label[i] == 1 ? -log(ans[i]) : -log(1.0 - ans[i]);
            if (ans[i] > 0.5 && test_label[i] == 1) correct++;
            else if (ans[i] < 0.5 && test_label[i] == 0) correct++;
        }
        std::cout << "total log likelihood = " << loss << " correct = " << std::setprecision(5)
                  << (float)correct / test_dataRow_cnt;
        printf(" auc = %.4f\n", Auc());
        if (savePath != "") {
            std::ofstream md(savePath);
            if (!md.is_open()) { std::cout << "save model open file error" << std::endl; exit(0); }
            for (auto v : ans) md << v << std::endl;
            md.close();
        }
    }
    std::vector<float> ans;

private:
    float Auc() {  // util/evaluator.h:51-104
        const size_t kHashLen = (1 << 24) - 1;
        std::vector<int> PosNum(kHashLen + 1, 0), NegNum(kHashLen + 1, 0);
        for (size_t i = 0; i < ans.size(); i++) {
            size_t index = ans[i] * kHashLen;
            if (test_label[i] == 1) PosNum[index]++; else NegNum[index]++;
        }
        float totPos = 0.0, totNeg = 0.0, totPosPrev = 0.0, totNegPrev = 0.0, auc = 0.0;
        for (int64_t idx = kHashLen; idx >= 0; --idx) {
            totPosPrev = totPos; totNegPrev = totNeg;
            totPos += PosNum[idx]; totNeg += NegNum[idx];
            auc += (totNeg > totNegPrev ? (totNeg - totNegPrev) : (totNegPrev - totNeg)) * (totPos + totPosPrev) / 2.0;
        }
        if (totPos > 0.0 && totNeg > 0.0) return auc / totPos / totNeg;
        return 0.0;
    }
    FM_Algo_Abst* fm;
    bool quirks_;
    size_t test_dataRow_cnt;
    std::vector<int64_t> row_ptr;
    std::vector<uint32_t> fid;
    std::vector<uint16_t> field;
    std::vector<float> val;
    std::vector<int32_t> test_label;
};

// ==========================================================================================================
// dl_algo_abst.h / train/layer/layer_abst.h / fullyconnLayer.h: the dense-layer surface
// ==========================================================================================================
// The reference drives these classes one SAMPLE at a time from a thread pool (dl_algo_abst.h:70-105): Predict(rid) ->
// Layer_Base::forward down the chain, BP(rid) -> backward up the chain, applyBP once per minibatch.  On the GPU the unit
// of work is the minibatch, so the same methods take the minibatch's rows at once (row-major [rows][dimension] floats)
// and lower to lctr_mlp_forward / lctr_mlp_backward / lctr_mlp_apply; names, call order, chaining through
// prevLayer / nextLayer, initialisation order of the rand() stream (fullyconnLayer.h:48-54) and the re-drawn dropout
// masks of applyBatchGradient (:200-202) are the reference's.
struct Sigmoid { static const int code = LCTR_ACT_SIGMOID; };
struct Tanh { static const int code = LCTR_ACT_TANH; };

class Layer_Base {  // layer_abst.h:25-83
public:
    Layer_Base(Layer_Base* _prevLayer, size_t _input_dimension, size_t _output_dimension)
        : input_dimension(_input_dimension), output_dimension(_output_dimension) {
        nextLayer = prevLayer = NULL;
        if (_prevLayer != NULL) {
            if (_prevLayer->output_dimension != this->input_dimension) { std::cout << "layer dimension mismatch" << std::endl; exit(1); }
            this->prevLayer = _prevLayer;
            _prevLayer->nextLayer = this;
            bInputLayer = false;
            printf("Init %zux%zu ", _input_dimension, _output_dimension);
        } else {
            bInputLayer = true;
            printf("Init Input %zux%zu ", _input_dimension, _output_dimension);
        }
    }
    virtual ~Layer_Base() {}
    // rows x input_dimension in, the chain's last output (rows x its output_dimension) back -- call on the input layer
    virtual std::vector<float>& forward(const std::vector<float>& prevLOutput, size_t rows) = 0;
    // rows x output_dimension deltas of the LAST layer in -- call on the output layer; walks back to the input layer
    virtual void backward(const std::vector<float>& outputDelta, size_t rows) = 0;
    virtual void applyBatchGradient() { if (nextLayer) nextLayer->applyBatchGradient(); }
    Layer_Base *nextLayer, *prevLayer;
    size_t input_dimension, output_dimension;
    bool bInputLayer;
};

template <typename ActivationFunction>
class Fully_Conn_Layer : public Layer_Base {  // fullyconnLayer.h:15-238
public:
    Fully_Conn_Layer(Layer_Base* _prevLayer, size_t _input_dimension, size_t _output_dimension)
        : Layer_Base(_prevLayer, _input_dimension, _output_dimension), needInputDelta(false), ctx(NULL), index(0) {
        weight = new float[input_dimension * output_dimension];
        bias = new float[output_dimension];
        dropout_mask = new float[output_dimension];
        for (size_t i = 0; i < output_dimension; i++) {  // init(), :48-54: bias, mask, then the row of weights
            bias[i] = 0.0;
            dropout_mask[i] = SampleBinary(GradientUpdater::__global_sparse_rate) ? 1. : 0.;
            for (size_t j = 0; j < input_dimension; j++) *getWeight(i, j) = UniformNumRand() - 0.5f;
        }
        if (_prevLayer) index = static_cast<Fully_Conn_Layer*>(_prevLayer)->index + 1;
        printf("Fully Connected Layer\n");
    }
    ~Fully_Conn_Layer() {
        delete[] weight; delete[] bias; delete[] dropout_mask;
        if (bInputLayer && ctx) lctr_destroy(ctx);
    }
    std::vector<float>& forward(const std::vector<float>& x, size_t rows) {
        if (!bInputLayer) { std::cout << "forward(): call on the input layer of the chain" << std::endl; exit(1); }
        ensure_ctx();
        Fully_Conn_Layer* last = this;
        while (last->nextLayer) last = static_cast<Fully_Conn_Layer*>(last->nextLayer);
        out_buf.resize(rows * last->output_dimension);
        LCTR_OK(lctr_mlp_forward(ctx, (int64_t)rows, x.data(), out_buf.data()));
        return out_buf;  // output layer returns wx + b without activator (:116)
    }
    void backward(const std::vector<float>& outputDelta, size_t rows) {
        Fully_Conn_Layer* first = this;
        while (first->prevLayer) first = static_cast<Fully_Conn_Layer*>(first->prevLayer);
        if (nextLayer || !first->ctx) { std::cout << "backward(): call on the output layer after forward()" << std::endl; exit(1); }
        first->input_delta.resize(rows * first->input_dimension);
        LCTR_OK(lctr_mlp_backward(first->ctx, (int64_t)rows, outputDelta.data(), first->needInputDelta ? first->input_delta.data() : NULL));
    }
    const std::vector<float>& inputDelta() const { return input_delta; }  // :189-192 (needInputDelta)
    void applyBatchGradient() {  // :194-206, on the input layer: updater, then every layer re-draws its mask in order
        if (bInputLayer) {
            ensure_ctx();
            LCTR_OK(lctr_mlp_apply(ctx, GradientUpdater::__global_minibatch_size));
        }
        for (size_t i = 0; i < output_dimension; i++) dropout_mask[i] = SampleBinary(GradientUpdater::__global_sparse_rate) ? 1. : 0.;
        Fully_Conn_Layer* first = this;
        while (first->prevLayer) first = static_cast<Fully_Conn_Layer*>(first->prevLayer);
        LCTR_OK(lctr_mlp_set_mask(first->ctx, (int)index, dropout_mask));
        if (nextLayer) nextLayer->applyBatchGradient();
    }
    // host copies of the parameters (pulled from the device on demand)
    void syncFromDevice() {
        Fully_Conn_Layer* first = this;
        while (first->prevLayer) first = static_cast<Fully_Conn_Layer*>(first->prevLayer);
        if (first->ctx) LCTR_OK(lctr_mlp_download(first->ctx, (int)index, weight, bias));
    }
    inline float* getWeight(size_t out_idx, size_t in_idx) const { return &weight[out_idx * input_dimension + in_idx]; }  // :211-216
    bool needInputDelta;
    float *weight, *bias, *dropout_mask;

private:
    void ensure_ctx() {  // the chain is complete once forward() is called: one device context for all its layers
        if (ctx) return;
        std::vector<Fully_Conn_Layer*> chain;
        for (Layer_Base* l = this; l; l = l->nextLayer) chain.push_back(static_cast<Fully_Conn_Layer*>(l));
        if (chain.size() < 2 || chain.size() > LCTR_MAX_LAYERS + 1 || chain.back()->output_dimension != 1) {
            std::cout << "Fully_Conn_Layer chain: 2.." << LCTR_MAX_LAYERS + 1 << " layers ending in one output" << std::endl;
            exit(1);
        }
        lctr_cfg cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.abi_version = LCTR_ABI_VERSION;
        cfg.model = LCTR_MODEL_NFM;       // dense chain on a factor_cnt-wide input; the embedding side stays unused
        cfg.feature_cnt = 1;
        cfg.factor_cnt = (uint32_t)input_dimension;
        cfg.learning_rate = GradientUpdater::__global_learning_rate;
        cfg.minibatch_size = GradientUpdater::__global_minibatch_size;
        cfg.n_hidden = (int32_t)chain.size() - 1;
        for (size_t l = 0; l + 1 < chain.size(); l++) cfg.hidden[l] = (uint32_t)chain[l]->output_dimension;
        cfg.activation = ActivationFunction::code;
        cfg.mlp_precision = LCTR_MLP_FP32;
        LCTR_OK(lctr_create(&cfg, &ctx));
        for (size_t l = 0; l < chain.size(); l++) {
            LCTR_OK(lctr_mlp_upload(ctx, (int)l, chain[l]->weight, chain[l]->bias));
            LCTR_OK(lctr_mlp_set_mask(ctx, (int)l, chain[l]->dropout_mask));
        }
    }
    lctr_ctx* ctx;  // owned by the input layer
    size_t index;   // position in the chain
    std::vector<float> out_buf, input_delta;
};

struct Logistic {};  // util/loss.h: gradient = pred - label on the sigmoid output
enum DL_Algo { DNN, CNN, RNN };

// dl_algo_abst.h:25-246.  Same constructor, members and Train() / validate() flow; Predict / BP take the minibatch's row
// ids at once.  `shuffle` (default true = the reference's random_shuffle per epoch, :62) can be switched off for parity runs.
template <typename LossFunction, typename ActivationFunction, typename OutputActivationFunction>
class DL_Algo_Abst {
public:
    DL_Algo_Abst(std::string dataPath, size_t _epoch, size_t _feature_cnt, size_t hidden_size, size_t _multiclass_output_cnt = 1)
        : shuffle(true), feature_cnt(_feature_cnt), multiclass_output_cnt(_multiclass_output_cnt), epoch(_epoch) {
        (void)hidden_size;
        if (_multiclass_output_cnt != 1) { std::cout << "the GPU dense path covers the single-output (CTR) case" << std::endl; exit(1); }
        this->dl_algo = DNN;
        loadDataRow(dataPath);
    }
    virtual ~DL_Algo_Abst() { for (size_t i = 0; i < network.size(); i++) delete network[i]; }
    virtual void initNetwork(size_t hidden_size) = 0;
    virtual const std::vector<float>& Predict(const std::vector<size_t>& rids, std::vector<std::vector<float> >& dataSet) = 0;
    virtual void BP(const std::vector<size_t>& rids, const std::vector<float>& grad) = 0;
    virtual void applyBP(size_t epoch) const = 0;
    void appendNNLayer(Layer_Base* layer) { network.push_back(layer); }

    void Train() {  // :53-134
        size_t batch_epoch = 0;
        const size_t mb = GradientUpdater::__global_minibatch_size;
        for (size_t p = 0; p < epoch; p++) {
            GradientUpdater::__global_bTraining = true;
            std::vector<size_t> inner_order(dataRow_cnt);
            for (size_t i = 0; i < dataRow_cnt; i++) inner_order[i] = i;
            if (shuffle) std::random_shuffle(inner_order.begin(), inner_order.end());
            for (size_t b = 0; b < dataRow_cnt; b += mb) {
                std::vector<size_t> rids(inner_order.begin() + b, inner_order.begin() + std::min(b + mb, dataRow_cnt));
                std::vector<float> pred = Predict(rids, dataSet);
                std::vector<float> grad(pred.size());
                for (size_t i = 0; i < pred.size(); i++) {
                    pred[i] = sigmoid_forward(pred[i]);            // outputActivFun.forward (:79)
                    grad[i] = pred[i] - (float)label[rids[i]];     // lossFun.gradient, Logistic (:91)
                }
                BP(rids, grad);
                applyBP(batch_epoch);
                validate(batch_epoch++);
            }
        }
    }
    void validate(size_t batch_epoch) {  // :136-176
        if (batch_epoch % 50 != 0) return;
        GradientUpdater::__global_bTraining = false;
        std::vector<size_t> all(dataRow_cnt);
        for (size_t i = 0; i < dataRow_cnt; i++) all[i] = i;
        std::vector<float> pred = Predict(all, dataSet);
        float loss = 0.0f;
        int correct = 0;
        for (size_t i = 0; i < dataRow_cnt; i++) {
            const float p = sigmoid_forward(pred[i]);
            // argmax over one output is index 0 (:150-154): "correct" counts label == 0 exactly like the reference
            if (label[i] == 0) correct++;
            loss += (label[i] == 1) ? -log(p) : -log(1.0f - p);
        }
        printf("Epoch %zu Loss = %f correct = %.3f\n", batch_epoch, loss, 1.0f * correct / dataRow_cnt);
        last_loss = loss;
        GradientUpdater::__global_bTraining = true;
    }
    virtual void loadDataRow(std::string dataPath) {  // :178-226, MNIST rows "label p0 p1 ..." (binary: label < 5 -> 0)
        dataSet.clear();
        std::ifstream fin_;
        std::string line;
        int nchar, y, val;
        size_t fid = 0;
        fin_.open(dataPath, std::ios::in);
        if (!fin_.is_open()) { std::cout << "open file error!" << std::endl; exit(1); }
        while (!fin_.eof()) {
            std::vector<float> tmp(feature_cnt, 0.f);
            getline(fin_, line);
            const char* pline = line.c_str();
            if (sscanf(pline, "%d%n", &y, &nchar) >= 1) {
                pline += nchar + 1;
                y = y < 5 ? 0 : 1;
                label.push_back(y);
                fid = 0;
                while (pline < line.c_str() + (int)line.length() && sscanf(pline, "%d%n", &val, &nchar) >= 1) {
                    pline += nchar + 1;
                    if (*pline == ',') pline += 1;
                    if (val != 0 && fid < feature_cnt) tmp[fid] = val / 255.0;
                    fid++;
                    if (fid > feature_cnt) break;
                }
                dataSet.push_back(tmp);
                if (dataSet.size() > 500) break;
            }
        }
        this->dataRow_cnt = this->dataSet.size();
        if (dataRow_cnt == 0 || label.size() != dataRow_cnt) { std::cout << "empty dataset" << std::endl; exit(1); }
    }
    bool shuffle;
    float last_loss;

protected:
    static float sigmoid_forward(float x) {  // util/activations.h:65-72
        if (x < -16.f) return 1e-7f;
        if (x > 16.f) return (float)(1.0 - 1e-7);
        return 1.0f / (1.0f + expf(-x));
    }
    DL_Algo dl_algo;
    std::vector<Layer_Base*> network;
    Layer_Base *inputLayer, *outputLayer;
    size_t feature_cnt, multiclass_output_cnt, dataRow_cnt;
    size_t epoch;
    std::vector<std::vector<float> > dataSet;
    std::vector<int> label;
};

// ==========================================================================================================
// distributed_algo_abst.h:86-340 -- Wide&Deep worker: one process per GPU instead of ZeroMQ workers + parameter servers
// ==========================================================================================================
// Same constructor (`<dataPath>_<rank>.csv`, :95-101), members and Train() / Predict() flow.  What the reference keeps
// on parameter-server processes -- the wide weights (scalar SGD, paramserver.h:295-300) and the per-feature tensors
// (tensor SGD, :232-237) -- lives in owner-sharded tables across the ranks' GPUs (owner = fid mod world) and moves
// over NVLink peer memory; every worker trains its OWN dense layers, as in the reference (:115-118, :279).
// Rank / world come from LIGHTCTR_B200_RANK / LIGHTCTR_B200_WORLD (the reference: `worker.Rank()` from its master); with
// world > 1 the CUDA-IPC handles and the global feature / field counts are exchanged through files in the directory
// LIGHTCTR_B200_RDV (any channel works: the blobs are opaque, see INTEGRATION.md).
class Distributed_Algo_Abst {
public:
    Distributed_Algo_Abst(std::string _dataPath, size_t _epoch_cnt) : epoch(_epoch_cnt), ctx(NULL), ds(NULL) {
        const char* er = getenv("LIGHTCTR_B200_RANK");
        const char* ew = getenv("LIGHTCTR_B200_WORLD");
        rank = er ? atoi(er) : 0;
        world = ew ? atoi(ew) : 1;
        std::stringstream ss;
        ss << _dataPath << "_" << rank << ".csv";
        loadDataRow(ss.str());
        L2Reg_ratio = 0.f;
        batch_size = GradientUpdater::__global_minibatch_size;
        if (world > 1) exchange_counts();
        // dense layers: input layer first, then the output layer (:115-117) -- the order of the rand() stream
        for (int l = 0; l < 2; l++) {
            const size_t in = l == 0 ? field_cnt * factor_dim : 50, out = l == 0 ? 50 : 1;
            layers.push_back(Fully_Conn_Layer_Host(in, out));
        }
        make_ctx();
    }
    ~Distributed_Algo_Abst() {
        if (ds) lctr_free_dataset(ds);
        if (ctx) lctr_destroy(ctx);
    }
    void Train() {  // :130-161
        GradientUpdater::__global_bTraining = true;
        std::vector<float> loss_curve, accuracy_curve;
        for (size_t i = 0; i < this->epoch; i++) {
            train_loss = 0;
            accuracy = 0;
            const size_t minibatch_epoch = (this->dataRow_cnt + this->batch_size - 1) / this->batch_size;
            for (size_t p = 0; p < minibatch_epoch; p++) {
                const size_t start_pos = p * batch_size;
                float l = 0, c = 0;
                LCTR_OK(lctr_train_step(ctx, 0, (int64_t)start_pos, (int64_t)std::min(start_pos + batch_size, this->dataRow_cnt), &l, &c));
                train_loss += l;
                accuracy += (size_t)c;
                for (size_t li = 0; li < layers.size(); li++) {  // applyBatchGradient re-draws the masks (:279)
                    layers[li].resample();
                    LCTR_OK(lctr_mlp_set_mask(ctx, (int)li, layers[li].mask.data()));
                }
            }
            printf("[Worker Train] epoch = %zu loss = %f accuracy = %f\n", i, train_loss, 1.0 * accuracy / dataRow_cnt);
            loss_curve.push_back(train_loss);
            accuracy_curve.push_back(1.0 * accuracy / dataRow_cnt);
        }
        for (size_t i = 0; i < this->epoch; i++) printf("%f(%.3f) ", loss_curve[i], accuracy_curve[i]);
        puts("");
        puts("Train Task Complete");
        GradientUpdater::__global_bTraining = false;
    }
    void Predict() {  // :163-174
        GradientUpdater::__global_bTraining = false;
        train_loss = 0;
        accuracy = 0;
        std::vector<float> p(dataRow_cnt);
        LCTR_OK(lctr_predict(ctx, 0, -1, p.data()));
        for (size_t rid = 0; rid < dataRow_cnt; rid++) {
            const float pCTR = p[rid];
            train_loss += (int)ds->label[rid] == 1 ? -log(pCTR) : -log(1.0 - pCTR);
            if (pCTR >= 0.5 && ds->label[rid] == 1) accuracy++;        // (>= here, > in the trainers: :239-243)
            else if (pCTR < 0.5 && ds->label[rid] == 0) accuracy++;
        }
        printf("[Worker Predict] loss = %f accuracy = %f\n", train_loss, 1.0 * accuracy / dataRow_cnt);
    }
    float last_loss() const { return train_loss; }
    size_t feature_cnt, field_cnt, dataRow_cnt;
    float L2Reg_ratio;
    static const size_t factor_dim = 4;  // :327
    std::vector<Fully_Conn_Layer_Host> layers;
    lctr_ctx* ctx;

private:
    void loadDataRow(std::string dataPath) {  // :283-318 (libffm rows; counts from the data)
        if (lctr_load_libffm(dataPath.c_str(), 0, 0, &ds) != 0) { std::cout << "open file error!" << std::endl; exit(1); }
        feature_cnt = ds->feature_cnt;
        field_cnt = 0;
        for (int64_t i = 0; i < ds->nnz; i++) field_cnt = std::max(field_cnt, (size_t)ds->field[i] + 1);
        dataRow_cnt = (size_t)ds->rows;
    }
    std::string rdv(const char* what, int r) const {
        const char* dir = getenv("LIGHTCTR_B200_RDV");
        if (!dir) { std::cout << "world > 1 needs LIGHTCTR_B200_RDV (a directory all ranks can write)" << std::endl; exit(1); }
        std::stringstream ss;
        ss << dir << "/" << what << "_" << r << ".bin";
        return ss.str();
    }
    void put(const char* what, const void* data, size_t bytes) const {
        const std::string path = rdv(what, rank), tmp = path + ".tmp";
        FILE* f = fopen(tmp.c_str(), "wb");
        if (!f || fwrite(data, 1, bytes, f) != bytes) { std::cout << "rendezvous write error" << std::endl; exit(1); }
        fclose(f);
        rename(tmp.c_str(), path.c_str());
    }
    void get(const char* what, int r, void* data, size_t bytes) const {
        const std::string path = rdv(what, r);
        for (int tries = 0; tries < 60000; tries++) {
            FILE* f = fopen(path.c_str(), "rb");
            if (f) {
                const size_t n = fread(data, 1, bytes, f);
                fclose(f);
                if (n == bytes) return;
            }
            struct timespec ts = {0, 1000000};
            nanosleep(&ts, NULL);
        }
        std::cout << "rendezvous timeout: " << path << std::endl;
        exit(1);
    }
    void exchange_counts() {  // the tables are sized for the largest id any rank has seen (the PS grows on demand)
        size_t mine[2] = {feature_cnt, field_cnt};
        put("counts", mine, sizeof(mine));
        for (int r = 0; r < world; r++) {
            size_t other[2];
            get("counts", r, other, sizeof(other));
            feature_cnt = std::max(feature_cnt, other[0]);
            field_cnt = std::max(field_cnt, other[1]);
        }
    }
    void make_ctx() {
        lctr_cfg cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.abi_version = LCTR_ABI_VERSION;
        cfg.model = LCTR_MODEL_WND;
        cfg.optimizer = LCTR_OPT_PS_SGD;  // ParamServer(UpdaterType::SGD), paramserver.h:49
        const char* dev = getenv("LIGHTCTR_B200_DEVICE");
        cfg.device = dev ? atoi(dev) : rank;
        cfg.feature_cnt = feature_cnt;
        cfg.field_cnt = (uint32_t)field_cnt;
        cfg.factor_cnt = (uint32_t)factor_dim;
        cfg.learning_rate = GradientUpdater::__global_learning_rate;
        cfg.l2_reg = L2Reg_ratio;
        cfg.minibatch_size = GradientUpdater::__global_minibatch_size;
        cfg.n_hidden = 1;
        cfg.hidden[0] = 50;
        cfg.activation = LCTR_ACT_TANH;  // Fully_Conn_Layer<Tanh> input layer (:115)
        cfg.mlp_precision = LCTR_MLP_FP32;
        cfg.rank = rank;
        cfg.world = world;
        cfg.max_nnz = (uint64_t)ds->nnz;
        LCTR_OK(lctr_create(&cfg, &ctx));
        // wide weights start at 0 (Value::initParam, :73-75), tensors at GaussRand() (TensorWrapper, paramserver.h:41-45);
        // drawn here per feature in id order, identically on every rank, after the layers' draws
        std::vector<float> W(feature_cnt, 0.f), E(feature_cnt * factor_dim);
        for (size_t i = 0; i < E.size(); i++) E[i] = GaussRand();
        LCTR_OK(lctr_upload_params(ctx, W.data(), E.data()));
        for (size_t l = 0; l < layers.size(); l++) {
            LCTR_OK(lctr_mlp_upload(ctx, (int)l, layers[l].weight.data(), layers[l].bias.data()));
            LCTR_OK(lctr_mlp_set_mask(ctx, (int)l, layers[l].mask.data()));
        }
        if (world > 1) {
            size_t n = 0;
            LCTR_OK(lctr_ipc_export(ctx, NULL, 0, &n));
            std::vector<char> mine(n), all((size_t)world * n);
            LCTR_OK(lctr_ipc_export(ctx, mine.data(), n, &n));
            put("ipc", mine.data(), n);
            for (int r = 0; r < world; r++) get("ipc", r, all.data() + (size_t)r * n, n);
            LCTR_OK(lctr_ipc_import(ctx, all.data(), n));
            char done = 1;  // every rank has mapped its peers before anybody's first key list goes out
            put("mapped", &done, 1);
            for (int r = 0; r < world; r++) get("mapped", r, &done, 1);
        }
        LCTR_OK(lctr_upload_batch(ctx, 0, ds->rows, ds->nnz, ds->row_ptr, ds->fid, ds->field, ds->val, ds->label));
    }
    size_t epoch, batch_size;
    int rank, world;
    float train_loss;
    size_t accuracy;
    lctr_dataset* ds;
};

}  // namespace lightctr_b200
#endif
