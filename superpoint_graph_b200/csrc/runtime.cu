// Runtime services of libspg_b200: error strings, launch accounting, memset.
#include <atomic>
#include <mutex>
#include <vector>

#include <stdlib.h>

#include "common.cuh"

namespace spg {

static const char* kKernelNames[K_COUNT] = {
    "ecc_vv_fwd",        "ecc_mat_fwd",        "ecc_generic_fwd",     "ecc_vv_bwd_w",
    "ecc_mat_bwd_w",     "ecc_generic_bwd_w",  "ecc_vv_bwd_x",        "ecc_mat_bwd_x",
    "ecc_generic_bwd_x", "gru_cell_fwd",       "gru_cell_bwd",        "gemm_f32",
    "gemm_splitk_reduce", "colstats_final",    "bn_fold",
    "affine_act",        "colsum_partial",     "colsum_final",        "act_bwd_reduce",
    "act_bwd_reduce_final", "act_bwd_apply",   "cloud_rows",          "segmax_fwd",
    "segmax_bwd",        "stn_apply_bwd",      "rows_scatter",        "rows_gather",
    "ce_loss",           "ce_loss_final",      "clamp_adam",          "tc_gemm_3xtf32",
    "tc_pack_weights",     "tc_dw_3xtf32",       "rnn_ecc_gru_fwd",     "rnn_ecc_gru_bwd",
    "cloud_build",       "confusion_count",    "tc_merge",
    "pointnet_fused_eval", "graph_build",
    "dropout_rng_next",  "dropout_fwd",        "dropout_mask",        "dropout_bwd_reduce",
    "dropout_bwd_reduce_final", "dropout_bwd_apply",
    "crf_fwd",           "crf_bwd",            "crf_softmax",
    "lstm_cell_fwd",     "lstm_cell_bwd",      "rnn_ecc_lstm_fwd",    "rnn_ecc_lstm_bwd",
    "gn_fwd",            "gn_bwd",             "gn_bwd_final",
    "lp_incidence",      "lp_dist_fwd",        "lp_dist_bwd",         "lp_loss_fwd",
    "lp_loss_bwd",       "lp_cc",              "lp_xpart",            "lp_seal",
    "lp_weights",        "lp_relax",           "lp_metrics",
    "lp_augment",        "lp_subgraph",        "lp_local_clouds",
    "geo_bounds",        "geo_grid",           "geo_knn",             "geo_geof",
    "sp_scan",           "sp_sort_keys",       "sp_points",           "sp_tets",
    "sp_pairs",          "sp_edges",
    "prune_bounds",      "prune_keys",         "prune_rows",          "prune_reduce",
    "cp_graph",          "cp_members",         "cp_kmeans",           "cp_centers",
    "cp_capacities",     "cp_maxflow",         "cp_colour",           "cp_activate",
    "cp_split",          "cp_merge",           "cp_energy",
    "dt_setup",          "dt_init",            "dt_nominate",         "dt_grow",
    "dt_check",          "dt_commit",          "dt_relocate",         "dt_output",
    "st_vor",            "st_cc",              "st_labels",           "st_select",
    "st_points",         "sb_select",          "sb_edges",
    "sb_draw",           "sb_perm",            "sb_flags",            "sb_cloud_draw",
};

struct Record {
    int kid;
    cudaEvent_t start, stop;
};

static std::atomic<long long> g_launches[K_COUNT];
static std::atomic<int> g_enabled{0};
static std::mutex g_mu;
static std::vector<Record> g_records;      // pending (not yet collected)
static std::vector<cudaEvent_t> g_free;    // recycled events
static double g_total_ms[K_COUNT];
static long long g_timed[K_COUNT];

static cudaEvent_t get_event() {
    if (!g_free.empty()) {
        cudaEvent_t e = g_free.back();
        g_free.pop_back();
        return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
}

static std::atomic<int> g_pdl{-1};  // -1: read SPG_PDL from the environment on first use (default on)

// mode 0: off; 1: every kernel; 2: every kernel except the persistent tensor-core kernels; 3: only the
// tensor-core GEMM and its merge companion
bool pdl_enabled(int kid) {
    int v = g_pdl.load(std::memory_order_relaxed);
    if (v < 0) {
        const char* e = getenv("SPG_PDL");
        v = e ? atoi(e) : 1;
        g_pdl.store(v, std::memory_order_relaxed);
    }
    const bool big = kid == K_TC_GEMM || kid == K_TC_DW || kid == K_POINTNET_FUSED;
    if (v == 2) return !big;
    if (v == 3) return kid == K_TC_GEMM || kid == K_TC_MERGE;
    return v != 0;
}

LaunchScope::LaunchScope(int kernel_id, cudaStream_t s) : kid(kernel_id), stream(s), slot(-1) {
    g_launches[kid].fetch_add(1, std::memory_order_relaxed);
    if (g_enabled.load(std::memory_order_relaxed)) {
        std::lock_guard<std::mutex> lk(g_mu);
        Record r;
        r.kid = kid;
        r.start = get_event();
        r.stop = get_event();
        cudaEventRecord(r.start, stream);
        g_records.push_back(r);
        slot = (int)g_records.size() - 1;
    }
}

LaunchScope::~LaunchScope() {
    if (slot >= 0) {
        std::lock_guard<std::mutex> lk(g_mu);
        if (slot < (int)g_records.size()) cudaEventRecord(g_records[slot].stop, stream);
    }
}

}  // namespace spg

using namespace spg;

extern "C" {

int spg_version(void) { return 100; }

int spg_set_pdl(int enabled) {
    g_pdl.store(enabled < 0 ? 0 : enabled, std::memory_order_relaxed);
    return SPG_OK;
}

const char* spg_error_string(int code) {
    if (code == SPG_OK) return "ok";
    if (code == SPG_E_BADARG) return "spg: bad argument (null pointer, negative size or bad flag)";
    if (code == SPG_E_UNSUPPORTED) return "spg: shape/dtype not supported by any kernel";
    if (code == SPG_E_ALIGN) return "spg: pointer or leading dimension misaligned";
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "spg: unknown error";
}

int spg_zero(void* ptr, int64_t bytes, spg_stream_t stream) {
    if (bytes < 0 || (!ptr && bytes > 0)) return SPG_E_BADARG;
    if (bytes == 0) return SPG_OK;
    return (int)cudaMemsetAsync(ptr, 0, (size_t)bytes, (cudaStream_t)stream);
}

int spg_prof_enable(int on) {
    g_enabled.store(on ? 1 : 0);
    return SPG_OK;
}

int spg_prof_reset(void) {
    std::lock_guard<std::mutex> lk(g_mu);
    for (auto& r : g_records) {
        g_free.push_back(r.start);
        g_free.push_back(r.stop);
    }
    g_records.clear();
    for (int i = 0; i < K_COUNT; ++i) {
        g_launches[i].store(0);
        g_total_ms[i] = 0.0;
        g_timed[i] = 0;
    }
    return SPG_OK;
}

int spg_prof_collect(void) {
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = SPG_OK;
    for (auto& r : g_records) {
        cudaError_t e = cudaEventSynchronize(r.stop);
        float ms = 0.f;
        if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, r.start, r.stop);
        if (e == cudaSuccess) {
            g_total_ms[r.kid] += ms;
            g_timed[r.kid] += 1;
        } else {
            rc = (int)e;
        }
        g_free.push_back(r.start);
        g_free.push_back(r.stop);
    }
    g_records.clear();
    return rc;
}

int spg_prof_num_kernels(void) { return K_COUNT; }

const char* spg_prof_kernel_name(int kernel_id) {
    if (kernel_id < 0 || kernel_id >= K_COUNT) return "";
    return kKernelNames[kernel_id];
}

int spg_prof_kernel_stats(int kernel_id, int64_t* launches, double* total_ms) {
    if (kernel_id < 0 || kernel_id >= K_COUNT) return SPG_E_BADARG;
    if (launches) *launches = g_launches[kernel_id].load();
    if (total_ms) *total_ms = g_total_ms[kernel_id];
    return SPG_OK;
}

int64_t spg_prof_total_launches(void) {
    long long t = 0;
    for (int i = 0; i < K_COUNT; ++i) t += g_launches[i].load();
    return t;
}

}  // extern "C"
