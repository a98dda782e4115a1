// pp_program: a recorded list of hot-path ops, replayed once per denoising step.
//
// The reference drives ~700-900 eager launches per UNet forward from Python
// (`for i, t in enumerate(timesteps)` loops, powerpaint/pipelines/pipeline_PowerPaint.py:988-1041,
// pipeline_PowerPaint_Brushnet_CA.py:1384-1466, pipeline_PowerPaint_ControlNet.py:1663-1741).
// Here the host plans the step once (tile selection, TMA tensor maps, buffer addresses),
// records it, and replays it — either as plain launches from C++ or as one CUDA graph whose
// per-step scalars (timestep, DDIM coefficients) are read from device tables indexed by a
// device-side step counter, so the same graph serves all steps.
#include <memory>
#include <vector>

#include "common.cuh"
#include "ops.h"

namespace pp {

enum OpKind {
    OP_GEMM, OP_ATTN, OP_GN, OP_LN, OP_UPSAMPLE, OP_ADD, OP_TIME_EMBED, OP_CFG_DDIM, OP_MEMSET, OP_SOFTMAX, OP_UNIPC, OP_EMBED, OP_CAUSAL_ATTN,
    OP_WINDOW_COPY, OP_TILE_BLEND, OP_SOLVER, OP_POOL_BROADCAST, OP_PLMS
};

struct LnArgs { const void* x; void* y; const float* gamma; const float* beta; int rows, c; float eps; };
struct UpArgs { const void* x; void* y; int nb, h, w, c, ho, wo; };
struct AddArgs { const void* a; const void* b; void* y; int64_t n; };
struct TeArgs { const float* timesteps; const int32_t* step_idx; void* out; int batch, dim; };
struct MsArgs { void* ptr; int64_t bytes; };
struct EmArgs { const int32_t* idx; const float* base; const float* ext; const float* pos; void* out; int rows, vocab, seq, dim; };
struct CaArgs { const void* qkv; void* out; int batch, seq, heads, d; float scale; };
struct SmArgs { const float* s; void* p; int64_t rows; int cols; int64_t ld_s, ld_p; };
struct WcArgs { const void* src; void* dst; int elem_bytes, channels; int64_t src_pix, dst_pix; const pp_window* windows; int count, max_pixels; };

struct Op {
    OpKind kind;
    union {
        GemmLaunch gemm;
        AttnLaunch attn;
        pp_gn_desc gn;
        LnArgs ln;
        UpArgs up;
        AddArgs add;
        TeArgs te;
        pp_cfg_ddim_desc ddim;
        MsArgs ms;
        SmArgs sm;
        EmArgs em;
        CaArgs ca;
        pp_unipc_desc unipc;
        WcArgs wc;
        pp_tile_blend_desc tb;
        pp_solver_desc solver;
        pp_pool_broadcast_desc pool;
        pp_plms_desc plms;
    };
    Op() { memset(this, 0, sizeof(*this)); }
};

}  // namespace pp

struct pp_program {
    std::vector<pp::Op> ops;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
};

namespace pp {

static int run_op(const Op& op, cudaStream_t s) {
    switch (op.kind) {
        case OP_GEMM: return gemm_launch(op.gemm, s);
        case OP_ATTN: return attn_launch(op.attn, s);
        case OP_GN: return group_norm_launch(op.gn, s);
        case OP_LN: return layer_norm_launch(op.ln.x, op.ln.y, op.ln.gamma, op.ln.beta, op.ln.rows, op.ln.c, op.ln.eps, s);
        case OP_UPSAMPLE: return upsample_nearest_launch(op.up.x, op.up.y, op.up.nb, op.up.h, op.up.w, op.up.c, op.up.ho, op.up.wo, s);
        case OP_ADD: return add_launch(op.add.a, op.add.b, op.add.y, op.add.n, s);
        case OP_TIME_EMBED: return time_embed_launch(op.te.timesteps, op.te.step_idx, op.te.out, op.te.batch, op.te.dim, s);
        case OP_CFG_DDIM: return cfg_ddim_launch(op.ddim, s);
        case OP_MEMSET:
            PP_CUDA_CHECK(cudaMemsetAsync(op.ms.ptr, 0, (size_t)op.ms.bytes, s));
            return PP_OK;
        case OP_UNIPC: return unipc_launch(op.unipc, s);
        case OP_EMBED: return embed_gather_launch(op.em.idx, op.em.base, op.em.ext, op.em.pos, op.em.out, op.em.rows, op.em.vocab, op.em.seq, op.em.dim, s);
        case OP_CAUSAL_ATTN: return causal_attention_small_launch(op.ca.qkv, op.ca.out, op.ca.batch, op.ca.seq, op.ca.heads, op.ca.d, op.ca.scale, s);
        case OP_SOFTMAX: return softmax_rows_launch(op.sm.s, op.sm.p, op.sm.rows, op.sm.cols, op.sm.ld_s, op.sm.ld_p, s);
        case OP_WINDOW_COPY: return window_copy_launch(op.wc.src, op.wc.dst, op.wc.elem_bytes, op.wc.channels, op.wc.src_pix,
                                                       op.wc.dst_pix, op.wc.windows, op.wc.count, op.wc.max_pixels, s);
        case OP_TILE_BLEND: return tile_blend_launch(op.tb, s);
        case OP_SOLVER: return solver_launch(op.solver, s);
        case OP_POOL_BROADCAST: return pool_broadcast_launch(op.pool, s);
        case OP_PLMS: return plms_launch(op.plms, s);
    }
    set_last_error("program: unknown op kind %d", (int)op.kind);
    return PP_ERR_INVALID;
}

static int launches_of(const Op& op) {
    switch (op.kind) {
        case OP_GN: return 2;  // stats + apply (the stats memset is a memset node, not a kernel)
        case OP_CFG_DDIM: return op.ddim.advance_step ? 2 : 1;
        case OP_UNIPC: return op.unipc.advance_step ? 2 : 1;
        case OP_SOLVER: return op.solver.advance_step ? 2 : 1;
        case OP_PLMS: return op.plms.advance_step ? 2 : 1;
        case OP_MEMSET: return 0;
        default: return 1;
    }
}

}  // namespace pp

#define PP_PROG_CHECK(p)                                                     \
    if (!(p)) {                                                              \
        pp::set_last_error("%s: null program", __func__);                    \
        return pp::PP_ERR_INVALID;                                           \
    }                                                                        \
    if ((p)->exec) {                                                         \
        pp::set_last_error("%s: program already built into a graph", __func__); \
        return pp::PP_ERR_INVALID;                                           \
    }

extern "C" {

pp_status pp_program_create(pp_program** out) {
    if (!out) { pp::set_last_error("pp_program_create: null out"); return pp::PP_ERR_INVALID; }
    *out = new pp_program();
    return pp::PP_OK;
}

void pp_program_destroy(pp_program* p) {
    if (!p) return;
    if (p->exec) cudaGraphExecDestroy(p->exec);
    if (p->graph) cudaGraphDestroy(p->graph);
    delete p;
}

pp_status pp_program_add_gemm(pp_program* p, const pp_gemm_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_gemm: null descriptor"); return pp::PP_ERR_INVALID; }
    pp::Op op;
    op.kind = pp::OP_GEMM;
    int rc = pp::gemm_prepare(*d, &op.gemm);
    if (rc) return rc;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_attention(pp_program* p, const pp_attn_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_attention: null descriptor"); return pp::PP_ERR_INVALID; }
    pp::Op op;
    op.kind = pp::OP_ATTN;
    int rc = pp::attn_prepare(*d, &op.attn);
    if (rc) return rc;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_group_norm(pp_program* p, const pp_gn_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_group_norm: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::group_norm_validate(*d);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_GN;
    op.gn = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_layer_norm(pp_program* p, const void* x, void* y, const float* gamma,
                                    const float* beta, int32_t rows, int32_t c, float eps) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(x && y && gamma && beta && rows > 0 && c > 0 && c % 8 == 0 && c <= 2048,
               "pp_program_add_layer_norm: invalid arguments (rows=%d c=%d)", rows, c);
    pp::Op op;
    op.kind = pp::OP_LN;
    op.ln = {x, y, gamma, beta, rows, c, eps};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_upsample2x(pp_program* p, const void* x, void* y, int32_t nb, int32_t h,
                                    int32_t w, int32_t c) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(x && y && nb > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "pp_program_add_upsample2x: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_UPSAMPLE;
    op.up = {x, y, nb, h, w, c, 2 * h, 2 * w};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_upsample_nearest(pp_program* p, const void* x, void* y, int32_t nb, int32_t h,
                                          int32_t w, int32_t c, int32_t ho, int32_t wo) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(x && y && nb > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0 && ho > 0 && wo > 0,
               "pp_program_add_upsample_nearest: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_UPSAMPLE;
    op.up = {x, y, nb, h, w, c, ho, wo};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_add(pp_program* p, const void* a, const void* b, void* y, int64_t n) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(a && b && y && n > 0 && n % 8 == 0, "pp_program_add_add: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_ADD;
    op.add = {a, b, y, n};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_time_embed(pp_program* p, const float* timesteps, const int32_t* step_idx,
                                    void* out, int32_t batch, int32_t dim) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(timesteps && out && batch > 0 && dim > 0 && dim % 2 == 0, "pp_program_add_time_embed: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_TIME_EMBED;
    op.te = {timesteps, step_idx, out, batch, dim};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_cfg_ddim(pp_program* p, const pp_cfg_ddim_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_cfg_ddim: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::cfg_ddim_validate(*d);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_CFG_DDIM;
    op.ddim = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_unipc(pp_program* p, const pp_unipc_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_unipc: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::unipc_validate(*d);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_UNIPC;
    op.unipc = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_solver_step(pp_program* p, const pp_solver_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_solver_step: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::solver_validate(*d);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_SOLVER;
    op.solver = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_plms_step(pp_program* p, const pp_plms_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_plms_step: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::plms_validate(*d);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_PLMS;
    op.plms = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_embed_gather(pp_program* p, const int32_t* idx, const float* base, const float* ext,
                                      const float* pos, void* out, int32_t rows, int32_t vocab, int32_t seq, int32_t dim) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(idx && base && pos && out && rows > 0 && vocab > 0 && seq > 0 && dim > 0 && dim % 4 == 0,
               "pp_program_add_embed_gather: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_EMBED;
    op.em = {idx, base, ext, pos, out, rows, vocab, seq, dim};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_causal_attention_small(pp_program* p, const void* qkv, void* out, int32_t batch, int32_t seq,
                                                int32_t heads, int32_t d, float scale) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(qkv && out && batch > 0 && heads > 0 && seq > 0 && seq <= 128 && (d == 8 || d == 16 || d == 32 || d == 64),
               "pp_program_add_causal_attention_small: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_CAUSAL_ATTN;
    op.ca = {qkv, out, batch, seq, heads, d, scale};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_memset(pp_program* p, void* ptr, int64_t bytes) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(ptr && bytes > 0, "pp_program_add_memset: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_MEMSET;
    op.ms = {ptr, bytes};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_softmax_rows(pp_program* p, const float* s, void* out, int64_t rows, int32_t cols,
                                      int64_t ld_s, int64_t ld_p) {
    PP_PROG_CHECK(p);
    PP_REQUIRE(s && out && rows > 0 && cols > 0 && cols <= 16384 && ld_s >= cols && ld_p >= cols,
               "pp_program_add_softmax_rows: invalid arguments");
    pp::Op op;
    op.kind = pp::OP_SOFTMAX;
    op.sm = {s, out, rows, cols, ld_s, ld_p};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_window_copy(pp_program* p, const void* src, void* dst, int32_t elem_bytes, int32_t channels,
                                     int64_t src_pix, int64_t dst_pix, const pp_window* windows, int32_t count,
                                     int32_t max_pixels) {
    PP_PROG_CHECK(p);
    int rc = pp::window_copy_validate(src, dst, elem_bytes, channels, src_pix, dst_pix, windows, count, max_pixels);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_WINDOW_COPY;
    op.wc = {src, dst, elem_bytes, channels, src_pix, dst_pix, windows, count, max_pixels};
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_tile_blend(pp_program* p, const pp_tile_blend_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_tile_blend: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::tile_blend_validate(*d);
    if (rc) return rc;
    PP_REQUIRE((int64_t)d->e_v * d->b_w + (int64_t)(d->b_h - d->e_v) * d->e_h > 0,
               "pp_program_add_tile_blend: the tile has no seam to blend");
    pp::Op op;
    op.kind = pp::OP_TILE_BLEND;
    op.tb = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

pp_status pp_program_add_pool_broadcast(pp_program* p, const pp_pool_broadcast_desc* d) {
    PP_PROG_CHECK(p);
    if (!d) { pp::set_last_error("pp_program_add_pool_broadcast: null descriptor"); return pp::PP_ERR_INVALID; }
    int rc = pp::pool_broadcast_validate(*d);
    if (rc) return rc;
    pp::Op op;
    op.kind = pp::OP_POOL_BROADCAST;
    op.pool = *d;
    p->ops.push_back(op);
    return pp::PP_OK;
}

int32_t pp_program_num_ops(const pp_program* p) { return p ? (int32_t)p->ops.size() : 0; }

int32_t pp_program_num_launches(const pp_program* p) {
    if (!p) return 0;
    int n = 0;
    for (const auto& op : p->ops) n += pp::launches_of(op);
    return n;
}

pp_status pp_program_run(pp_program* p, pp_stream stream) {
    if (!p) { pp::set_last_error("pp_program_run: null program"); return pp::PP_ERR_INVALID; }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    for (size_t i = 0; i < p->ops.size(); ++i) {
        int rc = pp::run_op(p->ops[i], s);
        if (rc) return rc;
    }
    return pp::PP_OK;
}

/* diagnostic: replay ops [first, first + count) as plain launches (bisecting a recorded step op by op) */
pp_status pp_program_run_range(pp_program* p, int32_t first, int32_t count, pp_stream stream) {
    if (!p) { pp::set_last_error("pp_program_run_range: null program"); return pp::PP_ERR_INVALID; }
    if (first < 0 || count < 0 || (size_t)first + (size_t)count > p->ops.size()) {
        pp::set_last_error("pp_program_run_range: [%d, %d) outside the %zu recorded ops", first, first + count, p->ops.size());
        return pp::PP_ERR_INVALID;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    for (int32_t i = first; i < first + count; ++i) {
        int rc = pp::run_op(p->ops[i], s);
        if (rc) return rc;
    }
    return pp::PP_OK;
}

pp_status pp_program_graph_build(pp_program* p, pp_stream stream) {
    if (!p) { pp::set_last_error("pp_program_graph_build: null program"); return pp::PP_ERR_INVALID; }
    if (p->exec) return pp::PP_OK;
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    // kernel attributes were set at record time, so launches are capturable as they are
    PP_CUDA_CHECK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    int rc = pp_program_run(p, stream);
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(s, &g);
    if (rc) {
        if (g) cudaGraphDestroy(g);
        return rc;
    }
    if (e != cudaSuccess) {
        pp::set_last_error("cudaStreamEndCapture failed: %s", cudaGetErrorString(e));
        return pp::PP_ERR_CUDA;
    }
    p->graph = g;
    PP_CUDA_CHECK(cudaGraphInstantiate(&p->exec, g, 0));
    return pp::PP_OK;
}

pp_status pp_program_graph_launch(pp_program* p, pp_stream stream) {
    if (!p || !p->exec) { pp::set_last_error("pp_program_graph_launch: graph not built"); return pp::PP_ERR_INVALID; }
    PP_CUDA_CHECK(cudaGraphLaunch(p->exec, reinterpret_cast<cudaStream_t>(stream)));
    return pp::PP_OK;
}

}  // extern "C"
