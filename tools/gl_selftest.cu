// Device-vs-host self test of the field arithmetic and the Poseidon2 permutation (development tool).
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -std=c++17 -Iinclude -o gl_selftest_bin tools/gl_selftest.cu   (then run ./gl_selftest_bin on the GPU)
#include <cstdio>
#include <vector>
#include "../deep-prove_b200/csrc/poseidon2.cuh"
#include "../deep-prove_b200/host/transcript.hpp"

__global__ void k_ops(const u64 *a, const u64 *b, u64 *out, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x; if (i >= n) return;
    u64 x = a[i], y = b[i], xc = gl_canon(x), yc = gl_canon(y);
    out[8 * i + 0] = gl_add(xc, yc);
    out[8 * i + 1] = gl_sub(xc, yc);
    out[8 * i + 2] = gl_mul(xc, yc);
    out[8 * i + 3] = gl_canon_weak(w_mul(x, y));
    gle e = e_mul(e_make(xc, yc), e_make(gl_canon(a[(i + 1) % n]), gl_canon(b[(i + 1) % n])));
    out[8 * i + 4] = e.c0; out[8 * i + 5] = e.c1;
    out[8 * i + 6] = gl_canon_weak(w_add(x, y));
    out[8 * i + 7] = gl_reduce160(x, y, (u32)(a[(i + 1) % n] & 0x7fffffffu));
}
__global__ void k_perm(const u64 *in, u64 *out, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x; if (i >= n) return;
    u64 s[8]; for (int k = 0; k < 8; k++) s[k] = in[8 * i + k];
    p2_permute(s);
    for (int k = 0; k < 8; k++) out[8 * i + k] = gl_canon_weak(s[k]);
}
__global__ void k_perm_lat(const u64 *in, u64 *out, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x; if (i >= n) return;
    u64 s[8]; for (int k = 0; k < 8; k++) s[k] = in[8 * i + k];
    p2_permute_lat(s);
    for (int k = 0; k < 8; k++) out[8 * i + k] = gl_canon_weak(s[k]);
}
__global__ void k_perm8(const u64 *in, u64 *out, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x; int h = i >> 3, l = i & 7; if (h >= n) return;
    u64 s = p2x8_permute(in[8 * h + l], l);
    out[8 * h + l] = gl_canon_weak(s);
}
static u64 sm(u64 &st) { u64 z = (st += 0x9E3779B97F4A7C15ULL); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL; z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL; return z ^ (z >> 31); }
int main() {
    const int n = 4096; u64 st = 1;
    std::vector<u64> a(n), b(n);
    for (int i = 0; i < n; i++) { a[i] = sm(st); b[i] = sm(st); }
    u64 edge[] = {0, 1, GL_P - 1, GL_P, GL_P + 1, ~0ULL, GL_EPS, GL_EPS + 1, 1ULL << 32, (1ULL << 63), ~0ULL - GL_EPS};
    int ne = sizeof(edge) / 8; for (int i = 0; i < ne; i++) for (int j = 0; j < ne; j++) { a[i * ne + j] = edge[i]; b[i * ne + j] = edge[j]; }
    p2_upload_constants((const u64 *)&DP_P2_EXT_RC[0][0][0], (const u64 *)DP_P2_INT_RC, (const u64 *)DP_P2_DIAG);
    u64 *da, *db, *dout; cudaMalloc(&da, n * 8); cudaMalloc(&db, n * 8); cudaMalloc(&dout, n * 64);
    cudaMemcpy(da, a.data(), n * 8, cudaMemcpyHostToDevice); cudaMemcpy(db, b.data(), n * 8, cudaMemcpyHostToDevice);
    k_ops<<<n / 128, 128>>>(da, db, dout, n);
    std::vector<u64> out(8 * n); cudaMemcpy(out.data(), dout, n * 64, cudaMemcpyDeviceToHost);
    const char *names[] = {"add", "sub", "mul", "w_mul", "emul.c0", "emul.c1", "w_add", "reduce160"};
    int bad[8] = {0};
    for (int i = 0; i < n; i++) {
        u64 x = a[i], y = b[i], xc = gl_canon(x), yc = gl_canon(y);
        u64 x2 = gl_canon(a[(i + 1) % n]), y2 = gl_canon(b[(i + 1) % n]);
        gle e = e_mul(e_make(xc, yc), e_make(x2, y2));
        u64 top = a[(i + 1) % n] & 0x7fffffffu;
        u64 exp[8] = {gl_add(xc, yc), gl_sub(xc, yc), gl_mul(xc, yc), gl_mul(xc, yc), e.c0, e.c1, gl_add(xc, yc), gl_reduce160(x, y, top)};
        for (int k = 0; k < 8; k++) if (out[8 * i + k] != exp[k]) { if (bad[k]++ < 3) printf("MISMATCH %s i=%d x=%llx y=%llx got=%llx exp=%llx\n", names[k], i, x, y, out[8 * i + k], exp[k]); }
    }
    for (int k = 0; k < 8; k++) printf("%-10s bad=%d\n", names[k], bad[k]);
    // permutation
    std::vector<u64> in(8 * n), pe(8 * n), p8(8 * n);
    for (auto &v : in) v = gl_canon(sm(st));
    for (int i = 0; i < 64; i++) for (int k = 0; k < 8; k++) in[8 * i + k] = ((i >> (k % 6)) & 1) ? GL_P - 1 - (u64)(i & 3) : (u64)(i & 7);   // extreme canonical words
    u64 *din, *dp; cudaMalloc(&din, n * 64); cudaMalloc(&dp, n * 64);
    cudaMemcpy(din, in.data(), n * 64, cudaMemcpyHostToDevice);
    k_perm<<<n / 128, 128>>>(din, dp, n); cudaMemcpy(pe.data(), dp, n * 64, cudaMemcpyDeviceToHost);
    k_perm8<<<n * 8 / 128, 128>>>(din, dp, n); cudaMemcpy(p8.data(), dp, n * 64, cudaMemcpyDeviceToHost);
    std::vector<u64> pl(8 * n);
    k_perm_lat<<<n / 128, 128>>>(din, dp, n); cudaMemcpy(pl.data(), dp, n * 64, cudaMemcpyDeviceToHost);
    int b1 = 0, b8 = 0, bl = 0;
    for (int i = 0; i < n; i++) {
        uint64_t s[8]; for (int k = 0; k < 8; k++) s[k] = in[8 * i + k];
        dp::Poseidon2::permute(s);
        for (int k = 0; k < 8; k++) { if (pe[8 * i + k] != s[k]) b1++; if (p8[8 * i + k] != s[k]) b8++; if (pl[8 * i + k] != s[k]) bl++; }
    }
    printf("permute bad=%d  permute_x8 bad=%d  permute_lat bad=%d  (cuda: %s)\n", b1, b8, bl, cudaGetErrorString(cudaDeviceSynchronize()));
    return 0;
}
