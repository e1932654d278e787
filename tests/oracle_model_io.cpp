// CHECKER -- TEST INFRASTRUCTURE ONLY.  The public IO of a model proof on the CPU restatement (oracle/): the model's output
// (zk_run) and the restated verifier run against an output the caller supplies, e.g. the one the device returned.  Built next to
// this file as libdp_oracle_model_io.so; ctypes view: tests/oracle_model_io.py.
#include "../oracle/zk_verify.hpp"
#include <string>

using namespace dpo;
static thread_local std::string g_err;

// a model given as the layer descriptor of dph_model_context_new (deep-prove_b200/models.py): 9 int64 per node {kind, 8 shape
// words}, weights in node order
static Model parse_model(const int64_t *desc, u32 n_nodes, const int64_t *data, u64 input_len) {
    Model m; m.input_len = input_len; const int64_t *w = data;
    for (u32 i = 0; i < n_nodes; i++) {
        const int64_t *d = desc + 9 * (size_t)i; Node n;
        switch (d[0]) {
        case 0: n.kind = OP_DENSE; n.nrows = d[1]; n.ncols = d[2]; n.weights.assign(w, w + n.nrows * n.ncols); w += n.nrows * n.ncols; n.bias.assign(w, w + n.nrows); w += n.nrows; break;
        case 1: n.kind = OP_REQUANT; n.rq.right_shift = d[1]; n.rq.fp_scale = d[2]; n.rq.fixed_point_multiplier = d[3]; n.rq.intermediate_bit_size = d[4]; break;
        case 2: n.kind = OP_RELU; break;
        case 3: { n.kind = OP_CONV; auto c = std::make_shared<ConvLayer>(); c->kw = d[1]; c->kx = d[2]; c->nw = d[3]; c->real_nw = d[4]; for (int k = 0; k < 3; k++) c->unpadded_out[k] = d[5 + k];
                  size_t fl = c->kw * c->kx * c->real_nw * c->real_nw; c->filter.assign(w, w + fl); w += fl; c->bias.assign(w, w + c->kw); w += c->kw; n.conv = c; break; }
        case 4: n.kind = OP_POOL; n.pool_c = d[1]; n.pool_h = d[2]; n.pool_w = d[3]; break;
        case 5: n.kind = OP_MATMUL; n.mm_r = d[1]; n.mm_k = d[2]; n.mm_c = d[3]; n.mm_t = d[4] != 0; n.mm_bias = d[5] != 0; n.weights.assign(w, w + n.mm_k * n.mm_c); w += n.mm_k * n.mm_c; if (n.mm_bias) { n.bias.assign(w, w + n.mm_c); w += n.mm_c; } break;
        default: throw std::runtime_error("unknown node kind");
        }
        m.nodes.push_back(n);
    }
    return m;
}

extern "C" {

const char *dpo_io_last_error() { return g_err.c_str(); }

// zk_run(m, input).back(): *out_len = its length; a null `out` only asks for the length, a `cap` below it is refused
int dpo_model_output(const int64_t *desc, u32 n_nodes, const int64_t *data, const int64_t *input, u64 input_len, int64_t *out, u64 cap, u64 *out_len) {
    try {
        Model m = parse_model(desc, n_nodes, data, input_len);
        std::vector<Element> y = zk_run(m, std::vector<Element>(input, input + input_len)).back();
        *out_len = y.size();
        if (!out) return 0;
        if (y.size() > cap) { g_err = "dpo_model_output: output buffer too small"; return 2; }
        memcpy(out, y.data(), 8 * y.size());
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

// Prove `input` on the checker, then verify the proof on a fresh transcript with the restated verifier against the CALLER's
// `output` (output_len elements) as the public output.  0 = accepted; 1 = rejected or not provable (dpo_io_last_error says why).
int dpo_model_verify_output(const int64_t *desc, u32 n_nodes, const int64_t *data, const int64_t *input, u64 input_len, const int64_t *output,
                            u64 output_len, const char *label) {
    try {
        Model m = parse_model(desc, n_nodes, data, input_len);
        std::vector<Element> in(input, input + input_len), out(output, output + output_len);
        ZkContext ctx = zk_context(m);
        Transcript tp(label);
        ModelProof p = zk_prove(ctx, in, tp);
        Transcript tv(label);
        zk_verify(ctx, in, out, p, tv);
        return 0;
    } catch (std::exception &e) { g_err = e.what(); return 1; }
}

}  // extern "C"
