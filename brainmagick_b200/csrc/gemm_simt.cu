// The FP32-FMA GEMM of gemm_simt.cuh: its kernel and launcher, one copy for every entry point that runs it.
#include "gemm_simt.cuh"

namespace bm {

__global__ void __launch_bounds__(GNT, 2) gemm_simt_kernel(const GemmP p) {
    __shared__ __align__(16) float As[2][GBK][GBM + GPAD];
    __shared__ __align__(16) float Bs[2][GBK][GBN + GPAD];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * GBM;
    const int seg = blockIdx.z / p.ksplit, kc = blockIdx.z - seg * p.ksplit;
    int zb, ze;
    if (p.seg_off) {
        zb = p.seg_off[seg];
        ze = p.seg_off[seg + 1];
    } else {
        zb = seg * p.zchunk;
        ze = min(p.Z, zb + p.zchunk);
    }
    const int kb = kc * p.kchunk, ke = min(p.K, kb + p.kchunk);
    const int nk = (ke - kb + GBK - 1) / GBK;
    const int total = max(0, ze - zb) * p.taps * nk;

    // column remap (GLU pairs column c with c + N/2 inside one tile)
    const int half = GBN / 2;
    const int Nh = p.N / 2;
    auto gcol = [&](int nn) -> int {
        if (p.glu) {
            int c = blockIdx.x * half + (nn < half ? nn : nn - half);
            if (c >= Nh) return -1;
            return nn < half ? c : Nh + c;
        }
        int n = blockIdx.x * GBN + nn;
        return n < p.N ? n : -1;
    };

    // loader element mapping (recomputed from tid inside the unrolled loops: keeps the kernel at <= 128 registers so
    // that two CTAs fit per SM, which is what hides the latency of the scalar tile loads)
    const int a_r0 = p.a_mcontig ? (tid & 127) : (tid >> 4), a_k0 = p.a_mcontig ? (tid >> 7) : (tid & 15);
    const int a_rs = p.a_mcontig ? 0 : 16, a_ks = p.a_mcontig ? 2 : 0;
    const int b_c0 = p.b_ncontig ? (tid & 127) : (tid >> 4), b_k0 = p.b_ncontig ? (tid >> 7) : (tid & 15);
    const int b_cs = p.b_ncontig ? 0 : 16, b_ks = p.b_ncontig ? 2 : 0;

    float ra[8], rb[8];
    auto load_tile = [&](int it) {
        int kt = it % nk;
        int r2 = it / nk;
        int tap = r2 % p.taps;
        int zi = zb + r2 / p.taps;
        if (p.zlist) zi = p.zlist[zi];
        int bz = p.bsel ? p.bsel[zi] : zi;
        const float* Ab = p.A + (long long)zi * p.lda_z;
        const float* Bb = p.B + (long long)bz * p.ldb_z + (long long)tap * p.ldb_tap;
        const int sh_m = p.a_shift_m[tap], sh_k = p.b_shift_k[tap];
        const int k0 = kb + kt * GBK;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int k = k0 + a_k0 + a_ks * i;
            int m = m0 + a_r0 + a_rs * i;
            int ms = m + sh_m;
            bool ok = (k < ke) && (m < p.M) && (ms >= 0) && (ms < p.M);
            ra[i] = ok ? __ldg(Ab + (long long)ms * p.lda_m + (long long)k * p.lda_k) : 0.f;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            int k = k0 + b_k0 + b_ks * i;
            int ks = k + sh_k;
            int n = gcol(b_c0 + b_cs * i);
            bool ok = (n >= 0) && (k < ke) && (ks >= 0) && (ks < p.K);
            rb[i] = ok ? __ldg(Bb + (long long)n * p.ldb_n + (long long)ks * p.ldb_k) : 0.f;
        }
    };
    auto store_tile = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            As[buf][a_k0 + a_ks * i][a_r0 + a_rs * i] = ra[i];
            Bs[buf][b_k0 + b_ks * i][b_c0 + b_cs * i] = rb[i];
        }
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    if (total > 0) {
        load_tile(0);
        store_tile(0);
    }
    __syncthreads();
    for (int it = 0; it < total; ++it) {
        const int cur = it & 1;
        if (it + 1 < total) load_tile(it + 1);
#pragma unroll
        for (int kk = 0; kk < GBK; ++kk) {
            float4 a0 = *reinterpret_cast<const float4*>(&As[cur][kk][ty * 4]);
            float4 a1 = *reinterpret_cast<const float4*>(&As[cur][kk][64 + ty * 4]);
            float4 b0 = *reinterpret_cast<const float4*>(&Bs[cur][kk][tx * 4]);
            float4 b1 = *reinterpret_cast<const float4*>(&Bs[cur][kk][64 + tx * 4]);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (it + 1 < total) store_tile(cur ^ 1);
        __syncthreads();
    }

    // ---------------- epilogue ----------------
    const long long dz = (long long)seg * p.ldd_z;
    int rows[8], cols[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        int r = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        rows[i] = r < p.M ? r : -1;
        cols[i] = gcol(i < 4 ? tx * 4 + i : 64 + tx * 4 + (i - 4));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (cols[j] < 0) continue;
        const float cs = p.colscale ? p.colscale[cols[j]] : 1.f;
        const float bs = (p.bias && kc == 0 && (!p.atomic || seg == 0)) ? p.bias[cols[j]] : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (rows[i] < 0) continue;
            float v = acc[i][j] * cs + bs;
            if (p.addend) v += p.addend[dz + (long long)rows[i] * p.ldd_m + (long long)cols[j] * p.ldd_n];
            acc[i][j] = v;
        }
    }
    if (p.stats) {
        // per-column sum / sumsq over this tile's valid rows -> fp64 atomics (BatchNorm batch statistics).  fp64 from the
        // first add: bn_finalize_kernel takes the variance as E[y^2] - E[y]^2, and fp32 sums of squares would lose it to
        // rounding once a channel's mean is ~100x its standard deviation.  The two [16][128] fp64 tables fit in As / Bs.
        double* red_s = reinterpret_cast<double*>(&As[0][0][0]);
        double* red_q = reinterpret_cast<double*>(&Bs[0][0][0]);
        static_assert(sizeof(As) >= 16 * GBN * sizeof(double) && sizeof(Bs) >= 16 * GBN * sizeof(double), "");
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            double s = 0.0, q = 0.0;
#pragma unroll
            for (int i = 0; i < 8; ++i)
                if (rows[i] >= 0 && cols[j] >= 0) { const double v = acc[i][j]; s += v; q = fma(v, v, q); }
            int nn = j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4);
            red_s[ty * GBN + nn] = s;
            red_q[ty * GBN + nn] = q;
        }
        __syncthreads();
        if (tid < GBN) {
            int n = gcol(tid);
            if (n >= 0) {
                double s = 0.0, q = 0.0;
#pragma unroll
                for (int r = 0; r < 16; ++r) { s += red_s[r * GBN + tid]; q += red_q[r * GBN + tid]; }
                atomicAdd(p.stats + n, s);
                atomicAdd(p.stats + p.N + n, q);
            }
        }
    }
    if (p.glu) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (cols[j] < 0) continue;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                if (rows[i] < 0) continue;
                float a = acc[i][j], g = acc[i][j + 4];
                if (p.D) {
                    p.D[dz + (long long)rows[i] * p.ldd_m + (long long)cols[j] * p.ldd_n] = a;
                    p.D[dz + (long long)rows[i] * p.ldd_m + (long long)cols[j + 4] * p.ldd_n] = g;
                }
                p.glu_out[(long long)seg * p.ldg_z + (long long)rows[i] * p.ldg_m + (long long)cols[j] * p.ldg_n] =
                    a * sigmoid_f(g);
            }
        }
        return;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (cols[j] < 0) continue;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            if (rows[i] < 0) continue;
            long long off = dz + (long long)rows[i] * p.ldd_m + (long long)cols[j] * p.ldd_n;
            float v = acc[i][j];
            if (p.aux) p.aux[off] = v;
            if (p.act == 1) v = gelu_f(v);
            if (p.atomic) atomicAdd(p.D + off, v);
            else p.D[off] = v;
        }
    }
}

cudaError_t launch_gemm(const GemmP& p, cudaStream_t st) {
    int gx = p.glu ? (p.N / 2 + GBN / 2 - 1) / (GBN / 2) : (p.N + GBN - 1) / GBN;
    int gy = (p.M + GBM - 1) / GBM;
    int gz = p.nseg * p.ksplit;
    if (gx <= 0 || gy <= 0 || gz <= 0) return cudaSuccess;
    if (gy > 65535 || gz > 65535) return cudaErrorInvalidConfiguration;
    GemmP q = p;
    if (q.kchunk <= 0) q.kchunk = q.K;
    dim3 grid(gx, gy, gz);
    gemm_simt_kernel<<<grid, GNT, 0, st>>>(q);
    ++g_launches;
    return cudaGetLastError();
}

}  // namespace bm
