// Batch inference without proving: the quantised model's outputs for many inputs at once, exactly as the witness path
// (witness.cu, conv.cu) computes them, for a user who wants the outputs or the failing inputs before paying for proofs.
//
// Every Dense, MatMul and Convolution input is 8-bit (the plan refuses any other), so int8 x int8 products accumulated in int32 are
// the prover's integers whenever 128 * sum|w| + |b| < 2^31 for each output row / channel, which the plan checks once.  These
// layers are one GEMM kernel on the tensor cores (mma.sync m16n8k32 s8 -> s32):
//   Dense   M = batch,            N = rows,     K = cols          A = the input tensor, B = the weights as stored ([rows][cols])
//   MatMul  M = batch * R,        N = C,        K = inner         B = the constant matrix laid out [C][K] once, at plan time
//   Conv    M = batch * nw^2,     N = kw,       K = the filter taps that are non-zero for some output channel (implicit GEMM:
//           A(m, k) is gathered from the input through a per-plan tap table; the FFT convolution's flat-index rule is reproduced:
//           tap (c, a, b) at output position p reads x[c][p + a*nw + b] when that index lies inside the channel, else 0)
// The epilogue adds the bias, clears a convolution's garbage positions, and applies a following Requant (and a Relu after it)
// with the witness kernels' own rules (quant.cuh), so a requantised layer stores int8 and its int32 accumulators never reach
// HBM.  A layer not followed by a Requant stores int32.  Requant / Relu / Maxpool nodes that are not fused run as small
// element-wise kernels.  Every tensor keeps the trace's padded layout ([C][n][n] for images), so the output is word for word the
// trace's.  Error bits are kept per input.
#include "common.cuh"
#include "quant.cuh"
#include <algorithm>

static constexpr u32 BM = 64, BN = 64, BK = 32;   // block tile (4 warps of 32 x 32) and the MMA's K

struct InferGemm {
    const int8_t *x; u64 x_ld;             // the input tensor of input b at x + b * x_ld
    const int8_t *w; const int *bias;      // w: [Np][Kp] int8, K-contiguous, zero-padded; bias [N] or null
    const int2 *taps;                      // Convolution: per k {channel offset + tap offset, tap offset}
    u32 M, N, Kp, m_per, a_rs;             // GEMM rows, m_per of them per input; Dense/MatMul row q of an input starts at q * a_rs
    void *y; u64 y_ld; u32 y_rs, y_cs;     // element (m, n) goes to y + (m / m_per) * y_ld + (m % m_per) * y_rs + n * y_cs
    int y_s8, conv, rq, relu;
    u32 nw_log, u0, u1, u2;                // Convolution: position q = i * nw + j is kept when n < u0 && i < u1 && j < u2
    RqRule r;
    u32 *err;                              // one error word per input
};

__device__ __forceinline__ void mma_s8(int (&d)[4], const u32 (&a)[4], const u32 (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ u32 pack4(int v0, int v1, int v2, int v3) {
    return (u32)(v0 & 255) | ((u32)(v1 & 255) << 8) | ((u32)(v2 & 255) << 16) | ((u32)v3 << 24);
}

// MODE 0: A rows read as 32-bit words (Dense, MatMul with K % 4 == 0); 1: byte by byte (MatMul otherwise); 2: Convolution gather.
// Fragment layouts: PTX ISA, mma.m16n8k32 with .s8 operands.
template <int MODE>
__global__ void __launch_bounds__(128) k_infer_gemm(InferGemm g) {
    const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gi = lane >> 2, ti = lane & 3;
    const u32 m0 = blockIdx.x * BM + (warp & 1) * 32, n0 = blockIdx.y * BN + (warp >> 1) * 32;
    const int8_t *row[4]; u32 pos[4];      // row r = 2 * mi + h is m0 + 16 mi + gi + 8 h (clamped: rows past M are never stored)
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const u32 m = min(m0 + (r >> 1) * 16 + gi + (r & 1) * 8, g.M - 1), b = m / g.m_per, q = m % g.m_per;
        row[r] = g.x + b * g.x_ld + (MODE == 2 ? 0 : (u64)q * g.a_rs);
        pos[r] = q;
    }
    int acc[2][4][4];
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int ni = 0; ni < 4; ni++)
#pragma unroll
            for (int c = 0; c < 4; c++) acc[mi][ni][c] = 0;
    for (u32 k0 = 0; k0 < g.Kp; k0 += BK) {
        u32 bf[4][2], af[2][4];
#pragma unroll
        for (int ni = 0; ni < 4; ni++) {
            const int8_t *wp = g.w + (u64)(n0 + ni * 8 + gi) * g.Kp + k0 + ti * 4;
            bf[ni][0] = __ldg((const u32 *)wp); bf[ni][1] = __ldg((const u32 *)(wp + 16));
        }
        int2 tap[8];
        if (MODE == 2) {
#pragma unroll
            for (int j = 0; j < 8; j++) tap[j] = __ldg(g.taps + k0 + ti * 4 + (j >> 2) * 16 + (j & 3));
        }
#pragma unroll
        for (int r = 0; r < 4; r++)
#pragma unroll
            for (int kh = 0; kh < 2; kh++) {     // register h + 2 kh of m-tile mi: row gi + 8h, columns 4 ti + 16 kh + 0..3
                u32 v;
                if (MODE == 0) v = *(const u32 *)(row[r] + k0 + ti * 4 + kh * 16);
                else if (MODE == 1) { const int8_t *p = row[r] + k0 + ti * 4 + kh * 16; v = pack4(p[0], p[1], p[2], p[3]); }
                else {
                    int e[4];
#pragma unroll
                    for (int j = 0; j < 4; j++) { const int2 t = tap[kh * 4 + j]; e[j] = pos[r] + (u32)t.y < g.m_per ? row[r][pos[r] + t.x] : 0; }
                    v = pack4(e[0], e[1], e[2], e[3]);
                }
                af[r >> 1][(r & 1) + 2 * kh] = v;
            }
#pragma unroll
        for (int mi = 0; mi < 2; mi++)
#pragma unroll
            for (int ni = 0; ni < 4; ni++) mma_s8(acc[mi][ni], af[mi], bf[ni]);
    }
    // epilogue: accumulator c of tile (mi, ni) is row m0 + 16 mi + gi + 8 (c >> 1), column n0 + 8 ni + 2 ti + (c & 1)
#pragma unroll
    for (int mi = 0; mi < 2; mi++)
#pragma unroll
        for (int c2 = 0; c2 < 2; c2++) {
            const u32 m = m0 + mi * 16 + gi + c2 * 8;
            if (m >= g.M) continue;
            const u32 b = m / g.m_per, q = m % g.m_per;
            u32 e = 0;
#pragma unroll
            for (int ni = 0; ni < 4; ni++)
#pragma unroll
                for (int c1 = 0; c1 < 2; c1++) {
                    const u32 n = n0 + ni * 8 + ti * 2 + c1;
                    if (n >= g.N) continue;
                    long long v = (long long)acc[mi][ni][c2 * 2 + c1] + (g.bias ? g.bias[n] : 0);
                    if (g.conv && !(n < g.u0 && (q >> g.nw_log) < g.u1 && (q & ((1u << g.nw_log) - 1)) < g.u2)) v = 0;
                    if (g.rq) v = rq_rule(v, g.r, e).out;
                    if (g.relu) v = relu_rule(v, e);
                    const u64 o = b * g.y_ld + (u64)q * g.y_rs + (u64)n * g.y_cs;
                    if (g.y_s8) ((int8_t *)g.y)[o] = (int8_t)v; else ((int *)g.y)[o] = (int)v;
                }
            if (e) atomicOr(g.err + b, e);
        }
}

// element-wise nodes over `total` = batch x len elements; tensors of input b start at b * ld
template <class T>
__global__ void k_infer_requant(const T *x, u64 x_ld, int8_t *y, u64 y_ld, u64 len, u64 total, RqRule r, u32 *err) {
    for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
        const u64 b = t / len, i = t % len;
        u32 e = 0;
        y[b * y_ld + i] = (int8_t)rq_rule(x[b * x_ld + i], r, e).out;
        if (e) atomicOr(err + b, e);
    }
}
template <class T>
__global__ void k_infer_relu(const T *x, u64 x_ld, T *y, u64 y_ld, u64 len, u64 total, u32 *err) {
    for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
        const u64 b = t / len, i = t % len;
        u32 e = 0;
        y[b * y_ld + i] = (T)relu_rule(x[b * x_ld + i], e);
        if (e) atomicOr(err + b, e);
    }
}
// Maxpool2D, kernel = stride = 2, on [C][H][W]
template <class T>
__global__ void k_infer_pool(const T *x, u64 x_ld, T *y, u64 y_ld, u32 C, u32 H, u32 W, u64 total, u32 *err) {
    const u64 len = (u64)C * (H / 2) * (W / 2);
    for (u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (u64)gridDim.x * blockDim.x) {
        const u64 b = t / len, oi = t % len;
        const u32 cc = (u32)(oi % (W / 2)), r = (u32)((oi / (W / 2)) % (H / 2)), c = (u32)(oi / ((u64)(W / 2) * (H / 2)));
        const T *xb = x + b * x_ld + ((u64)c * H + 2 * r) * W + 2 * cc;
        const long long v[4] = {xb[0], xb[W], xb[1], xb[W + 1]};
        const long long mx = max(max(v[0], v[1]), max(v[2], v[3]));
        u32 e = 0;
        for (int k = 0; k < 4; k++) pool_rule(mx - v[k], e);
        y[b * y_ld + oi] = (T)mx;
        if (e) atomicOr(err + b, e);
    }
}

enum InferStageKind { GEMM, REQUANT, RELU, POOL };
struct InferTensor { bool s8; u64 len, ld; u64 bytes() const { return ld * (s8 ? 1 : 4); } };   // per input; ld rounded up to 32 elements
struct InferStage {
    InferStageKind kind; InferGemm g{};           // GEMM: everything but the tensor and error pointers
    int mode = 0; u32 C = 0, H = 0, W = 0;  // GEMM load mode; Maxpool shape
};

static int plan_fail(u32 id, const char *what, const std::string &msg) { return dp_fail(DP_ERR_INVALID, "dp_infer_plan: node " + std::to_string(id) + " (" + what + "): " + msg); }
static u64 round_up(u64 v, u64 a) { return (v + a - 1) / a * a; }

struct dp_infer {
    std::vector<InferTensor> t;        // t[s] is stage s's input, t.back() the model output
    std::vector<InferStage> s;
    std::vector<void *> dev;      // weights, biases and tap tables
    ~dp_infer() { for (void *p : dev) cudaFree(p); }
};

template <class V> static int upload(dp_infer *p, const std::vector<V> &v, const V **out) {
    *out = nullptr;
    if (v.empty()) return DP_OK;
    void *d = nullptr;
    DP_CUDA(cudaMalloc(&d, sizeof(V) * v.size()));
    p->dev.push_back(d);
    DP_CUDA(cudaMemcpy(d, v.data(), sizeof(V) * v.size(), cudaMemcpyHostToDevice));
    *out = (const V *)d;
    return DP_OK;
}

extern "C" {

int dp_infer_plan(const dp_infer_node *nodes, uint32_t n_nodes, uint64_t input_len, dp_infer **out) {
    DP_REQUIRE_CTX();
    DP_CHECK(out && (nodes || n_nodes == 0) && input_len > 0, DP_ERR_INVALID, "dp_infer_plan: null argument or empty input");
    *out = nullptr;
    static const char *NAMES[6] = {"Dense", "Requant", "Relu", "Convolution", "Maxpool", "MatMul"};
    std::unique_ptr<dp_infer> p(new dp_infer());
    p->t.push_back({true, input_len, round_up(input_len, 32)});
    bool eight = true;                    // the current tensor holds 8-bit values (the model input, or a Requant output since)
    for (u32 id = 0; id < n_nodes; id++) {
        const dp_infer_node &nd = nodes[id];
        DP_CHECK(nd.kind <= 5, DP_ERR_INVALID, "dp_infer_plan: node " + std::to_string(id) + ": unknown kind");
        const char *name = NAMES[nd.kind];
        const InferTensor cur = p->t.back();
        auto rq_params = [&](const dp_infer_node &r, u32 rid, RqRule &rule) {
            if (r.shift < 1 || r.shift > 62 || r.clamp_size < 1 || r.clamp_size > 62 || r.intermediate_bits > 62)
                return plan_fail(rid, "Requant", "shift and clamping size must lie in 1..62, intermediate bits in 0..62");
            rule = RqRule{r.shift, r.clamp_size, (long long)r.multiplier, 1LL << r.intermediate_bits};
            return DP_OK;
        };
        InferStage st;
        if (nd.kind == 1) {
            st.kind = REQUANT;
            if (int e = rq_params(nd, id, st.g.r)) return e;
            p->t.push_back({true, cur.len, round_up(cur.len, 32)});
            eight = true;
        } else if (nd.kind == 2) {
            st.kind = RELU;
            p->t.push_back(cur);
        } else if (nd.kind == 4) {
            st.kind = POOL; st.C = nd.dims[0]; st.H = nd.dims[1]; st.W = nd.dims[2];
            if ((u64)st.C * st.H * st.W != cur.len || st.H % 2 || st.W % 2 || st.H == 0 || st.W == 0) return plan_fail(id, name, "shape does not match its input");
            const u64 len = (u64)st.C * (st.H / 2) * (st.W / 2);
            p->t.push_back({cur.s8, len, round_up(len, 32)});
        } else {                          // Dense (0), Convolution (3), MatMul (5): one GEMM
            if (!eight) return plan_fail(id, name, "its input is not 8-bit (neither the model input nor a Requant output, optionally through Relu / Maxpool)");
            InferGemm &g = st.g; st.kind = GEMM;
            u64 N = 0, K = 0, out_len = 0;
            std::vector<int8_t> w; std::vector<int> bias; std::vector<int2> taps;
            std::vector<long long> wsrc;  // the weights as B[n][k], before the range checks
            const int64_t *bsrc = nd.bias;
            if (nd.kind == 0) {
                N = nd.dims[0]; K = nd.dims[1];
                if (K != cur.len || N == 0) return plan_fail(id, name, "ncols does not match its input");
                wsrc.assign(nd.weights, nd.weights + N * K);
                g.m_per = 1; g.a_rs = 0; g.y_rs = 0; g.y_cs = 1; out_len = N;
                st.mode = 0;
            } else if (nd.kind == 5) {
                const u64 R = nd.dims[0], KK = nd.dims[1], C = nd.dims[2]; const bool tr = nd.dims[3] != 0;
                if (R * KK != cur.len || C == 0 || R == 0) return plan_fail(id, name, "shape does not match its input");
                N = C; K = KK; wsrc.resize(N * K);
                for (u64 n = 0; n < N; n++) for (u64 k = 0; k < K; k++) wsrc[n * K + k] = tr ? nd.weights[n * K + k] : nd.weights[k * C + n];
                g.m_per = (u32)R; g.a_rs = (u32)K; g.y_rs = (u32)C; g.y_cs = 1; out_len = R * C;
                st.mode = K % 4 == 0 ? 0 : 1;
            } else {
                const u64 kw = nd.dims[0], kx = nd.dims[1], nw = nd.dims[2], rn = nd.dims[3];
                if (kx * nw * nw != cur.len || kw == 0 || rn == 0 || (nw & (nw - 1)) || cur.len > (u64)INT32_MAX) return plan_fail(id, name, "shape does not match its input");
                // a filter wider than the image has taps (b >= nw) that the FFT convolution drops and this gather would wrap into the
                // next row; the prover refuses such a layer (dp_pad_rows), so the plan does too
                if (rn > nw) return plan_fail(id, name, "filter width " + std::to_string(rn) + " exceeds the padded image width " + std::to_string(nw));
                const u64 P = nw * nw, T = kx * rn * rn;
                // keep the taps (c, a, b) with a non-zero weight for some output channel
                std::vector<u64> keep;
                for (u64 k = 0; k < T; k++) { bool nz = false; for (u64 o = 0; o < kw && !nz; o++) nz = nd.weights[o * T + k] != 0; if (nz) keep.push_back(k); }
                N = kw; K = keep.size(); wsrc.resize(N * K);
                for (u64 o = 0; o < N; o++) for (u64 k = 0; k < K; k++) wsrc[o * K + k] = nd.weights[o * T + keep[k]];
                for (u64 k : keep) { const u64 c = k / (rn * rn), a = (k / rn) % rn, b = k % rn, d = a * nw + b; taps.push_back(make_int2((int)(c * P + d), (int)std::min<u64>(d, P))); }
                taps.resize(round_up(K, BK), make_int2(0, (int)P));   // padding taps: never inside the channel
                g.m_per = (u32)P; g.y_rs = 1; g.y_cs = (u32)P; out_len = kw * P;
                g.conv = 1; g.u0 = nd.dims[4]; g.u1 = nd.dims[5]; g.u2 = nd.dims[6]; while ((1ULL << g.nw_log) < nw) g.nw_log++;
                st.mode = 2;
            }
            // exactness: every weight int8, every bias int32, and 128 * sum|w| + |b| <= 2^31 - 1 on each output row / channel
            const u64 Np = round_up(N, BN), Kp = round_up(K, BK);
            w.assign(Np * Kp, 0);
            for (u64 n = 0; n < N; n++) {
                long long s = 0;
                for (u64 k = 0; k < K; k++) {
                    const long long v = wsrc[n * K + k];
                    if (v < -128 || v > 127) return plan_fail(id, name, "weight " + std::to_string(v) + " outside [-128, 127]");
                    w[n * Kp + k] = (int8_t)v; s += v < 0 ? -v : v;
                }
                const long long b = bsrc ? bsrc[n] : 0;
                if (b < INT32_MIN || b > INT32_MAX) return plan_fail(id, name, "bias " + std::to_string(b) + " outside int32");
                if (128 * s + (b < 0 ? -b : b) > (long long)INT32_MAX)
                    return plan_fail(id, name, "output " + std::to_string(n) + " can exceed int32 (128 * sum|w| + |b| > 2^31 - 1)");
                if (bsrc) bias.push_back((int)b);
            }
            g.N = (u32)N; g.Kp = (u32)Kp;
            if (int e = upload(p.get(), w, &g.w)) return e;
            if (int e = upload(p.get(), bias, &g.bias)) return e;
            if (int e = upload(p.get(), taps, &g.taps)) return e;
            // a following Requant, and a Relu after that, run in the epilogue
            if (id + 1 < n_nodes && nodes[id + 1].kind == 1) {
                if (int e = rq_params(nodes[id + 1], id + 1, g.r)) return e;
                g.rq = 1; id++;
                if (id + 1 < n_nodes && nodes[id + 1].kind == 2) { g.relu = 1; id++; }
            }
            g.y_s8 = g.rq;
            eight = g.rq != 0;
            p->t.push_back({g.y_s8 != 0, out_len, round_up(out_len, 32)});
        }
        p->s.push_back(st);
    }
    *out = p.release();
    return DP_OK;
}

int dp_infer_run(dp_infer *p, const int64_t *inputs, uint32_t n, int64_t *outputs, uint32_t *err_bits) {
    DP_REQUIRE_CTX();
    DP_CHECK(p && inputs && outputs && err_bits && n > 0, DP_ERR_INVALID, "dp_infer_run: null argument or no inputs");
    cudaStream_t st = dp_ctx().stream;
    const InferTensor &ti = p->t.front(), &to = p->t.back();
    u64 buf_bytes = 0, max_rows = 1;      // per input: the largest tensor (two of them alternate), the most GEMM rows
    for (const InferTensor &t : p->t) buf_bytes = std::max(buf_bytes, t.bytes());
    for (const InferStage &s : p->s) if (s.kind == GEMM) max_rows = std::max<u64>(max_rows, s.g.m_per);
    size_t free_b = 0, total_b = 0;
    DP_CUDA(cudaMemGetInfo(&free_b, &total_b));
    const u64 per_input = 2 * buf_bytes + 4;
    u64 chunk = std::min<u64>({(u64)n, (u64)DP_INFER_MAX_CHUNK, (u64)(free_b / 2) / per_input, (u64)INT32_MAX / max_rows});
    DP_CHECK(chunk > 0, DP_ERR_CUDA, "dp_infer_run: not enough free device memory for one input");
    void *buf[2] = {nullptr, nullptr}; u32 *err = nullptr; int8_t *h_in = nullptr; void *h_out = nullptr; u32 *h_err = nullptr;
    struct Release {
        void **buf; u32 **err; int8_t **hi; void **ho; u32 **he;
        ~Release() { cudaFree(buf[0]); cudaFree(buf[1]); cudaFree(*err); cudaFreeHost(*hi); cudaFreeHost(*ho); cudaFreeHost(*he); }
    } release{buf, &err, &h_in, &h_out, &h_err};
    for (void *&b : buf) DP_CUDA(cudaMalloc(&b, chunk * buf_bytes + 64));   // + 64: the GEMM's unguarded reads past a MatMul row
    DP_CUDA(cudaMalloc((void **)&err, 4 * chunk));
    DP_CUDA(cudaMallocHost((void **)&h_in, chunk * ti.ld));
    DP_CUDA(cudaMallocHost(&h_out, chunk * to.bytes()));
    DP_CUDA(cudaMallocHost((void **)&h_err, 4 * chunk));
    std::vector<u32> bad(chunk);
    for (u64 c0 = 0; c0 < n; c0 += chunk) {
        const u64 nb = std::min<u64>(chunk, n - c0);
        for (u64 j = 0; j < nb; j++) {    // an input outside the 8-bit domain is computed as zeros and flagged (bit 16)
            const int64_t *x = inputs + (c0 + j) * ti.len; int8_t *h = h_in + j * ti.ld;
            bad[j] = 0;
            for (u64 i = 0; i < ti.len; i++) { if (x[i] < -128 || x[i] > 127) bad[j] = 16; h[i] = (int8_t)x[i]; }
            if (bad[j]) memset(h, 0, ti.len);
            memset(h + ti.len, 0, ti.ld - ti.len);
        }
        DP_CUDA(cudaMemcpyAsync(buf[0], h_in, nb * ti.ld, cudaMemcpyHostToDevice, st));
        DP_CUDA(cudaMemsetAsync(err, 0, 4 * nb, st));
        for (size_t si = 0; si < p->s.size(); si++) {
            const InferStage &s = p->s[si]; const InferTensor &a = p->t[si], &y = p->t[si + 1];
            void *x = buf[si & 1], *o = buf[(si + 1) & 1];
            const u64 total = nb * y.len;
            const int grid = dp_grid_for(total, 256, 8);
            if (s.kind == GEMM) {
                InferGemm g = s.g;
                g.x = (const int8_t *)x; g.x_ld = a.ld; g.y = o; g.y_ld = y.ld; g.err = err; g.M = (u32)(nb * g.m_per);
                const dim3 grid2((g.M + BM - 1) / BM, (g.N + BN - 1) / BN);
                DpProfScope prof("k_infer_gemm", nb * (a.bytes() + y.bytes()) + (u64)grid2.y * BN * g.Kp, 2ull * g.M * g.N * g.Kp);
                if (s.mode == 0) DP_CUDA(dp_launch(k_infer_gemm<0>, grid2, 128, 0, st, g));
                else if (s.mode == 1) DP_CUDA(dp_launch(k_infer_gemm<1>, grid2, 128, 0, st, g));
                else DP_CUDA(dp_launch(k_infer_gemm<2>, grid2, 128, 0, st, g));
            } else if (s.kind == REQUANT) {
                if (a.s8) DP_CUDA(dp_launch(k_infer_requant<int8_t>, grid, 256, 0, st, (const int8_t *)x, a.ld, (int8_t *)o, y.ld, y.len, total, s.g.r, err));
                else DP_CUDA(dp_launch(k_infer_requant<int>, grid, 256, 0, st, (const int *)x, a.ld, (int8_t *)o, y.ld, y.len, total, s.g.r, err));
            } else if (s.kind == RELU) {
                if (a.s8) DP_CUDA(dp_launch(k_infer_relu<int8_t>, grid, 256, 0, st, (const int8_t *)x, a.ld, (int8_t *)o, y.ld, y.len, total, err));
                else DP_CUDA(dp_launch(k_infer_relu<int>, grid, 256, 0, st, (const int *)x, a.ld, (int *)o, y.ld, y.len, total, err));
            } else {
                if (a.s8) DP_CUDA(dp_launch(k_infer_pool<int8_t>, grid, 256, 0, st, (const int8_t *)x, a.ld, (int8_t *)o, y.ld, s.C, s.H, s.W, total, err));
                else DP_CUDA(dp_launch(k_infer_pool<int>, grid, 256, 0, st, (const int *)x, a.ld, (int *)o, y.ld, s.C, s.H, s.W, total, err));
            }
        }
        DP_CUDA(cudaMemcpyAsync(h_out, buf[p->s.size() & 1], nb * to.bytes(), cudaMemcpyDeviceToHost, st));
        DP_CUDA(cudaMemcpyAsync(h_err, err, 4 * nb, cudaMemcpyDeviceToHost, st));
        DP_CUDA(dp_stream_sync(st));
        for (u64 j = 0; j < nb; j++) {
            int64_t *yo = outputs + (c0 + j) * to.len;
            if (to.s8) { const int8_t *h = (const int8_t *)h_out + j * to.ld; for (u64 i = 0; i < to.len; i++) yo[i] = h[i]; }
            else { const int *h = (const int *)h_out + j * to.ld; for (u64 i = 0; i < to.len; i++) yo[i] = h[i]; }
            err_bits[c0 + j] = h_err[j] | bad[j];
        }
    }
    return DP_OK;
}

int dp_infer_free(dp_infer *p) {
    delete p;
    return DP_OK;
}

}  // extern "C"
