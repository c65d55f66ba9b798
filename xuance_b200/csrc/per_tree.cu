// K5 prioritized-replay segment trees: insert / stratified sample / priority update.
// Trees are tiny relative to HBM (2 trees x 2*cap floats per env; 1 MB per env at cap = 65536) and stay
// L2-resident; the kernels are latency-bound pointer walks, so they are organised around warps:
// one CTA per env, per-sample lanes walking the tree, warp shuffles for the per-env reductions, and a
// level-synchronous rebuild for batched updates.  All node arithmetic is IEEE float32 with explicit
// round-to-nearest intrinsics (no FMA contraction) so that results are bit-identical to the float32 oracle.
#include "xb_common.cuh"

// ---- float32 pow bit-identical to glibc 2.39 powf (sysdeps/ieee754/flt-32/e_powf.c; algorithm and tables from
// ARM Optimized Routines: powf_log2_data.c, exp2f_data.c).  numpy's `np.float32 ** python_float` - what the
// reference's PER buffer evaluates (memory_tools.py:547,596) - calls exactly this libm routine, so the device
// restates it in double arithmetic with the same tables, polynomial order and FMA contraction.
__constant__ double POWF_LOG2_TAB[16][2] = {
    {0x1.661ec79f8f3bep+0, -0x1.efec65b963019p-2},
    {0x1.571ed4aaf883dp+0, -0x1.b0b6832d4fca4p-2},
    {0x1.49539f0f010b0p+0, -0x1.7418b0a1fb77bp-2},
    {0x1.3c995b0b80385p+0, -0x1.39de91a6dcf7bp-2},
    {0x1.30d190c8864a5p+0, -0x1.01d9bf3f2b631p-2},
    {0x1.25e227b0b8ea0p+0, -0x1.97c1d1b3b7af0p-3},
    {0x1.1bb4a4a1a343fp+0, -0x1.2f9e393af3c9fp-3},
    {0x1.12358f08ae5bap+0, -0x1.960cbbf788d5cp-4},
    {0x1.0953f419900a7p+0, -0x1.a6f9db6475fcep-5},
    {0x1.0000000000000p+0, 0x0.0p+0},
    {0x1.e608cfd9a47acp-1, 0x1.338ca9f24f53dp-4},
    {0x1.ca4b31f026aa0p-1, 0x1.476a9543891bap-3},
    {0x1.b2036576afce6p-1, 0x1.e840b4ac4e4d2p-3},
    {0x1.9c2d163a1aa2dp-1, 0x1.40645f0c6651cp-2},
    {0x1.886e6037841edp-1, 0x1.88e9c2c1b9ff8p-2},
    {0x1.767dcf5534862p-1, 0x1.ce0a44eb17bccp-2},
};
__constant__ unsigned long long EXP2F_TAB[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull,
};
__device__ __forceinline__ float powf_libm(float x, float y) {
    uint32_t ix = __float_as_uint(x);
    if (ix - 0x00800000u >= 0x7f800000u - 0x00800000u) {   // zero, subnormal, negative, inf or nan
        if (ix == 0u || ix >= 0x7f800000u) return powf(x, y);  // zero/negative/inf/nan: not on the PER path
        // subnormal: normalised as glibc does, x * 2^23 with the exponent lowered by 23 (it goes negative; the
        // unsigned wrap cancels in iz = ix - top below)
        ix = __float_as_uint(__fmul_rn(x, 0x1p23f)) & 0x7fffffffu;
        ix -= 23u << 23;
    }
    // log2(x) = log1p(z/c - 1)/ln2 + log2(c) + k
    const uint32_t tmp = ix - 0x3f330000u;
    const int i = (tmp >> 19) & 15;
    const uint32_t top = tmp & 0xff800000u;
    const uint32_t iz = ix - top;
    const int k = (int32_t)top >> 23;
    const double invc = POWF_LOG2_TAB[i][0], logc = POWF_LOG2_TAB[i][1];
    const double z = (double)__uint_as_float(iz);
    const double A0 = 0x1.27616c9496e0bp-2, A1 = -0x1.71969a075c67ap-2, A2 = 0x1.ec70a6ca7baddp-2,
                 A3 = -0x1.7154748bef6c8p-1, A4 = 0x1.71547652ab82bp+0;
    double r = __fma_rn(z, invc, -1.0);
    const double y0 = __dadd_rn(logc, (double)k);
    double r2 = __dmul_rn(r, r);
    double yy = __fma_rn(A0, r, A1);
    const double pp = __fma_rn(A2, r, A3);
    const double r4 = __dmul_rn(r2, r2);
    double q = __fma_rn(A4, r, y0);
    q = __fma_rn(pp, r2, q);
    yy = __fma_rn(yy, r4, q);
    const double ylogx = __dmul_rn((double)y, yy);
    if (fabs(ylogx) >= 126.0) {   // glibc's special cases; the rest of this range takes the exp2 path below
        if (ylogx > 0x1.fffffffd1d571p+6) return __uint_as_float(0x7f800000u);   // x^y rounds to inf
        if (ylogx <= -150.0) return 0.f;                                          // x^y rounds to 0
        if (ylogx < -149.0) return 0x1p-149f;                                     // glibc's __math_may_uflowf
    }
    // exp2(ylogx): x = k/N + r, N = 32
    const double SHIFT = 0x1.8p+47;
    double kd = __dadd_rn(ylogx, SHIFT);
    const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
    kd = __dsub_rn(kd, SHIFT);
    r = __dsub_rn(ylogx, kd);
    unsigned long long t = EXP2F_TAB[ki & 31];
    t += ki << 47;
    const double sc = __longlong_as_double((long long)t);
    const double C0 = 0x1.c6af84b912394p-5, C1 = 0x1.ebfce50fac4f3p-3, C2 = 0x1.62e42ff0c52d6p-1;
    const double zz = __fma_rn(C0, r, C1);
    r2 = __dmul_rn(r, r);
    double o = __fma_rn(C2, r, 1.0);
    o = __fma_rn(zz, r2, o);
    o = __dmul_rn(o, sc);
    return (float)o;
}

__device__ __forceinline__ float pow_alpha(float p, float alpha) { return powf_libm(p, alpha); }

// test hook: out[i] = powf_libm(x[i], y)
__global__ void powf_libm_kernel(const float *__restrict__ x, float y, float *__restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = powf_libm(x[i], y);
}
extern "C" int xb_powf_libm(const float *x, float y, float *out, int64_t n, void *stream) {
    if (!x || !out || n <= 0) return XB_EINVAL;
    powf_libm_kernel<<<(int)((n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184), 256, 0, (cudaStream_t)stream>>>(x, y, out, n);
    return xb_launch_status();
}

// ---------------------------------------------------------------- insert
__global__ void __launch_bounds__(32) per_insert_kernel(float *__restrict__ sum_tree, float *__restrict__ min_tree,
                                                        const float *__restrict__ max_prio, int N, int cap, int ptr,
                                                        float alpha) {
    const int env = blockIdx.x * blockDim.x + threadIdx.x;
    if (env >= N) return;
    float *st = sum_tree + (int64_t)env * 2 * cap;
    float *mt = min_tree + (int64_t)env * 2 * cap;
    const float leaf = pow_alpha(max_prio[env], alpha);
    int n = ptr + cap;
    st[n] = leaf;
    mt[n] = leaf;
    for (n >>= 1; n >= 1; n >>= 1) {
        st[n] = __fadd_rn(st[2 * n], st[2 * n + 1]);
        const float l = mt[2 * n], r = mt[2 * n + 1];
        mt[n] = (r < l) ? r : l;  // Python min(l, r): r only if strictly smaller
    }
}

extern "C" int xb_per_insert(float *sum_tree, float *min_tree, float *max_prio, int N, int cap, int ptr, float alpha,
                             void *stream) {
    if (!sum_tree || !min_tree || !max_prio || N <= 0 || cap <= 0 || (cap & (cap - 1)) || ptr < 0 || ptr >= cap)
        return XB_EINVAL;
    per_insert_kernel<<<(N + 31) / 32, 32, 0, (cudaStream_t)stream>>>(sum_tree, min_tree, max_prio, N, cap, ptr, alpha);
    return xb_launch_status();
}

// ---------------------------------------------------------------- sample
// reduce(0, end_incl) with the reference recursion's association: v[L1] + (v[L2] + (v[L3] + ...)).
__device__ float prefix_reduce_sum(const float *__restrict__ t, int cap, int end_incl) {
    float spine[33];
    int depth = 0;
    int node = 1, ns = 0, ne = cap - 1;
    while (true) {
        if (end_incl == ne) {
            spine[depth++] = t[node];
            break;
        }
        int mid = (ns + ne) >> 1;
        if (end_incl <= mid) {
            node = 2 * node;
            ne = mid;
        } else {
            spine[depth++] = t[2 * node];  // whole left child
            node = 2 * node + 1;
            ns = mid + 1;
        }
    }
    float acc = spine[depth - 1];
    for (int i = depth - 2; i >= 0; --i) acc = __fadd_rn(spine[i], acc);
    return acc;
}

__global__ void __launch_bounds__(256) per_sample_kernel(const float *__restrict__ sum_tree,
                                                         const float *__restrict__ min_tree,
                                                         const float *__restrict__ u, int cap, int size, int k,
                                                         int64_t S, float spb, int64_t *__restrict__ step_out,
                                                         int64_t *__restrict__ flat_out, double *__restrict__ w_out) {
    const int env = blockIdx.x;
    const float *st = sum_tree + (int64_t)env * 2 * cap;
    const float *mt = min_tree + (int64_t)env * 2 * cap;
    __shared__ float sh_seg, sh_maxw, sh_total;
    if (threadIdx.x == 0) {
        // p_total = sum(0, size-1): END-EXCLUSIVE -> inclusive range [0, size-2]   (memory_tools.py:520)
        int end = size - 1;
        if (end < 0) end += cap;
        end -= 1;
        float p_total = (end >= 0) ? prefix_reduce_sum(st, cap, end) : 0.f;
        sh_seg = __fdiv_rn(p_total, (float)k);
        const float total = st[1];
        const float p_min = __fdiv_rn(mt[1], total);
        sh_maxw = __fmul_rn(p_min, spb);
        sh_total = total;
    }
    __syncthreads();
    const float seg = sh_seg, total = sh_total, maxw = sh_maxw;
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        float mass = __fadd_rn(__fmul_rn(u[(int64_t)env * k + j], seg), __fmul_rn((float)j, seg));
        int n = 1;
        while (n < cap) {
            const float left = st[2 * n];
            if (left > mass) {
                n = 2 * n;
            } else {
                mass = __fsub_rn(mass, left);
                n = 2 * n + 1;
            }
        }
        const int step = n - cap;
        const float p_s = __fdiv_rn(st[n], total);
        const float w = __fdiv_rn(__fmul_rn(p_s, spb), maxw);
        step_out[(int64_t)env * k + j] = step;
        flat_out[(int64_t)env * k + j] = (int64_t)env * S + step;
        w_out[(int64_t)env * k + j] = (double)w;
    }
}

extern "C" int xb_per_sample(const float *sum_tree, const float *min_tree, const float *u, int N, int cap, int size,
                             int k, int64_t S, float size_pow_neg_beta, int64_t *step_out, int64_t *flat_out,
                             double *w_out, void *stream) {
    if (!sum_tree || !min_tree || !u || !step_out || !flat_out || !w_out) return XB_EINVAL;
    if (N <= 0 || cap <= 0 || (cap & (cap - 1)) || k <= 0 || size <= 0 || size > cap) return XB_EINVAL;
    per_sample_kernel<<<N, 256, 0, (cudaStream_t)stream>>>(sum_tree, min_tree, u, cap, size, k, S, size_pow_neg_beta,
                                                           step_out, flat_out, w_out);
    return xb_launch_status();
}

// ---------------------------------------------------------------- update
// One CTA per env.  Sequential semantics of the reference (later duplicates overwrite earlier ones, every
// write re-derives its ancestors) are reproduced by: (1) last-writer-wins leaf resolution, (2) recomputing the
// touched ancestors level by level - an internal node is always op(children), so the final tree is a pure
// function of the final leaves.
__global__ void __launch_bounds__(256) per_update_kernel(float *__restrict__ sum_tree, float *__restrict__ min_tree,
                                                         float *__restrict__ max_prio, const int64_t *__restrict__ idx,
                                                         const float *__restrict__ prio, int cap, int k, float alpha) {
    const int env = blockIdx.x;
    float *st = sum_tree + (int64_t)env * 2 * cap;
    float *mt = min_tree + (int64_t)env * 2 * cap;
    const int64_t *my_idx = idx + (int64_t)env * k;
    const float *my_p = prio + (int64_t)env * k;
    __shared__ float sh_max[8];
    float local_max = 0.f;
    // (1) leaves: item j writes unless a later item targets the same leaf
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        float p = my_p[j];
        if (p == 0.f) p = __fadd_rn(p, 1e-8f);
        local_max = fmaxf(local_max, p);
        const int64_t leaf = my_idx[j];
        bool last = true;
        for (int j2 = j + 1; j2 < k; ++j2)
            if (my_idx[j2] == leaf) {
                last = false;
                break;
            }
        if (last) {
            const float v = pow_alpha(p, alpha);
            st[leaf + cap] = v;
            mt[leaf + cap] = v;
        }
    }
    // max_priority[i] = max(max_priority[i], p) over the batch
    local_max = fmaxf(local_max, __shfl_xor_sync(0xffffffffu, local_max, 16));
    local_max = fmaxf(local_max, __shfl_xor_sync(0xffffffffu, local_max, 8));
    local_max = fmaxf(local_max, __shfl_xor_sync(0xffffffffu, local_max, 4));
    local_max = fmaxf(local_max, __shfl_xor_sync(0xffffffffu, local_max, 2));
    local_max = fmaxf(local_max, __shfl_xor_sync(0xffffffffu, local_max, 1));
    if ((threadIdx.x & 31) == 0) sh_max[threadIdx.x >> 5] = local_max;
    __syncthreads();
    if (threadIdx.x == 0) {
        float m = max_prio[env];
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m = fmaxf(m, sh_max[w]);
        max_prio[env] = m;
    }
    // (2) ancestors, level by level (duplicates recompute the same value: benign)
    for (int shift = 1; (cap >> shift) >= 1; ++shift) {
        __syncthreads();
        for (int j = threadIdx.x; j < k; j += blockDim.x) {
            const int n = (int)((my_idx[j] + cap) >> shift);
            st[n] = __fadd_rn(st[2 * n], st[2 * n + 1]);
            const float l = mt[2 * n], r = mt[2 * n + 1];
            mt[n] = (r < l) ? r : l;
        }
    }
}

extern "C" int xb_per_update(float *sum_tree, float *min_tree, float *max_prio, const int64_t *idx, const float *prio,
                             int N, int cap, int k, float alpha, void *stream) {
    if (!sum_tree || !min_tree || !max_prio || !idx || !prio) return XB_EINVAL;
    if (N <= 0 || cap <= 0 || (cap & (cap - 1)) || k <= 0) return XB_EINVAL;
    per_update_kernel<<<N, 256, 0, (cudaStream_t)stream>>>(sum_tree, min_tree, max_prio, idx, prio, cap, k, alpha);
    return xb_launch_status();
}
