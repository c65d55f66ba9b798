// K1 store, K2 GAE scan, K3 gathers (rows / observations / scalar fields + advantage normalisation).
// HBM-bound byte movers: 16-byte vector accesses, 1-D bulk-async (TMA unit) staging through shared memory
// for whole observation rows, persistent grids sized to the SM count.
#include "xb_common.cuh"

// =====================================================================================================
// K1  xb_rollout_store
// =====================================================================================================
// grid.x = N * chunks_per_row (+ scalar blocks); each thread moves 16 B (or 4 B tail words).
__global__ void __launch_bounds__(256) store_rows_kernel(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                                         int64_t row_bytes, int N, int T, int t, bool vec16,
                                                         float *__restrict__ sdst, const float *__restrict__ ssrc,
                                                         int F, int row_blocks) {
    if ((int)blockIdx.x >= row_blocks) {  // scalar fields: dst[f][n][t] = src[f][n]
        int i = (blockIdx.x - row_blocks) * blockDim.x + threadIdx.x;
        if (i < F * N) {
            int f = i / N, n = i - f * N;
            sdst[((int64_t)f * N + n) * T + t] = ssrc[i];
        }
        return;
    }
    const int64_t per_row = vec16 ? row_bytes / 16 : row_bytes / 4;
    const int64_t total = per_row * N;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)row_blocks * blockDim.x) {
        int64_t n = i / per_row, c = i - n * per_row;
        if (vec16) {
            uint4 v = ldg_stream16(src + n * row_bytes + c * 16);
            stg_stream16(dst + (n * T + t) * row_bytes + c * 16, v);
        } else {
            uint32_t v = *reinterpret_cast<const uint32_t *>(src + n * row_bytes + c * 4);
            *reinterpret_cast<uint32_t *>(dst + (n * T + t) * row_bytes + c * 4) = v;
        }
    }
}

extern "C" int xb_rollout_store(void *rows_dst, const void *rows_src, int64_t row_bytes, float *scal_dst,
                                const float *scal_src, int F, int N, int T, int t, void *stream) {
    if (N <= 0 || T <= 0 || t < 0 || t >= T || F < 0) return XB_EINVAL;
    if ((rows_dst == nullptr) != (rows_src == nullptr)) return XB_EINVAL;
    if (F > 0 && (!scal_dst || !scal_src)) return XB_EINVAL;
    int row_blocks = 0;
    bool vec16 = false;
    if (rows_dst) {
        if (row_bytes <= 0 || (row_bytes & 3)) return XB_EALIGN;
        vec16 = (row_bytes % 16 == 0) && xb_aligned(rows_dst, 16) && xb_aligned(rows_src, 16);
        if (!vec16 && (!xb_aligned(rows_dst, 4) || !xb_aligned(rows_src, 4))) return XB_EALIGN;
        int64_t items = (vec16 ? row_bytes / 16 : row_bytes / 4) * N;
        int64_t want = (items + 255) / 256;
        int64_t cap = (int64_t)xb_sm_count() * 8;
        row_blocks = (int)(want < cap ? want : cap);
        if (row_blocks < 1) row_blocks = 1;
    }
    int scal_blocks = F > 0 ? (F * N + 255) / 256 : 0;
    if (row_blocks + scal_blocks == 0) return XB_OK;
    store_rows_kernel<<<row_blocks + scal_blocks, 256, 0, (cudaStream_t)stream>>>(
        (uint8_t *)rows_dst, (const uint8_t *)rows_src, row_bytes, N, T, t, vec16, scal_dst, scal_src, F, row_blocks);
    return xb_launch_status();
}

// xb_rollout_store_at: the same store with a per-row step index step[n] read on the device (rows whose step is outside
// [0, T) are left alone).  A separate kernel so that xb_rollout_store's instructions stay as they are.
__global__ void __launch_bounds__(256) store_rows_at_kernel(uint8_t *__restrict__ dst, const uint8_t *__restrict__ src,
                                                            int64_t row_bytes, int N, int T,
                                                            const int32_t *__restrict__ step, bool vec16,
                                                            float *__restrict__ sdst, const float *__restrict__ ssrc,
                                                            int F, int row_blocks) {
    if ((int)blockIdx.x >= row_blocks) {
        int i = (blockIdx.x - row_blocks) * blockDim.x + threadIdx.x;
        if (i < F * N) {
            int f = i / N, n = i - f * N;
            const int t = step[n];
            if (t >= 0 && t < T) sdst[((int64_t)f * N + n) * T + t] = ssrc[i];
        }
        return;
    }
    const int64_t per_row = vec16 ? row_bytes / 16 : row_bytes / 4;
    const int64_t total = per_row * N;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)row_blocks * blockDim.x) {
        int64_t n = i / per_row, c = i - n * per_row;
        const int t = step[n];
        if (t < 0 || t >= T) continue;
        if (vec16) {
            uint4 v = ldg_stream16(src + n * row_bytes + c * 16);
            stg_stream16(dst + (n * T + t) * row_bytes + c * 16, v);
        } else {
            uint32_t v = *reinterpret_cast<const uint32_t *>(src + n * row_bytes + c * 4);
            *reinterpret_cast<uint32_t *>(dst + (n * T + t) * row_bytes + c * 4) = v;
        }
    }
}

extern "C" int xb_rollout_store_at(void *rows_dst, const void *rows_src, int64_t row_bytes, float *scal_dst,
                                   const float *scal_src, int F, int N, int T, const int32_t *step, void *stream) {
    if (N <= 0 || T <= 0 || F < 0 || !step) return XB_EINVAL;
    if ((rows_dst == nullptr) != (rows_src == nullptr)) return XB_EINVAL;
    if (F > 0 && (!scal_dst || !scal_src)) return XB_EINVAL;
    int row_blocks = 0;
    bool vec16 = false;
    if (rows_dst) {
        if (row_bytes <= 0 || (row_bytes & 3)) return XB_EALIGN;
        vec16 = (row_bytes % 16 == 0) && xb_aligned(rows_dst, 16) && xb_aligned(rows_src, 16);
        if (!vec16 && (!xb_aligned(rows_dst, 4) || !xb_aligned(rows_src, 4))) return XB_EALIGN;
        int64_t items = (vec16 ? row_bytes / 16 : row_bytes / 4) * N;
        int64_t want = (items + 255) / 256;
        int64_t cap = (int64_t)xb_sm_count() * 8;
        row_blocks = (int)(want < cap ? want : cap);
        if (row_blocks < 1) row_blocks = 1;
    }
    int scal_blocks = F > 0 ? (F * N + 255) / 256 : 0;
    if (row_blocks + scal_blocks == 0) return XB_OK;
    store_rows_at_kernel<<<row_blocks + scal_blocks, 256, 0, (cudaStream_t)stream>>>(
        (uint8_t *)rows_dst, (const uint8_t *)rows_src, row_bytes, N, T, step, vec16, scal_dst, scal_src, F,
        row_blocks);
    return xb_launch_status();
}

// =====================================================================================================
// K2  xb_gae_scan : one warp per env, reverse inclusive scan of affine maps x -> a*x + b over the T steps.
// =====================================================================================================
// A_t = delta_t + c_t * A_{t+1}.  Map f_t(x) = c_t*x + delta_t ; suffix composition F_t = f_t o f_{t+1} o ... ;
// A_t = F_t(0) = offset part.  Each lane owns V consecutive steps (vector loads), composes them serially, then a
// 5-step shuffle scan composes across lanes (from the high lanes down), tiles are chained through a carry.
template <typename R>
struct Affine {
    R a, b;
};  // x -> a*x + b
template <typename R>
__device__ __forceinline__ Affine<R> compose(const Affine<R> &f, const Affine<R> &g) {  // f o g
    return {f.a * g.a, f.a * g.b + f.b};
}
template <typename R>
__device__ __forceinline__ R shfl_down_t(R v, int d);
template <>
__device__ __forceinline__ float shfl_down_t<float>(float v, int d) { return __shfl_down_sync(0xffffffffu, v, d); }
template <>
__device__ __forceinline__ double shfl_down_t<double>(double v, int d) { return __shfl_down_sync(0xffffffffu, v, d); }

template <typename R, bool GAE, int V, bool VEC>
__global__ void __launch_bounds__(128) gae_scan_kernel(const float *__restrict__ rew, const float *__restrict__ val,
                                                       const float *__restrict__ term,
                                                       const uint8_t *__restrict__ seg_end,
                                                       const float *__restrict__ boot,
                                                       const int32_t *__restrict__ covered, float *__restrict__ adv,
                                                       float *__restrict__ ret, int N, int T, float gamma, float lam) {
    const int lane = threadIdx.x & 31;
    const int env = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (env >= N) return;
    const int64_t base = (int64_t)env * T;
    const int cov = covered ? covered[env] : T;
    const float gl = gamma * lam;
    const int TILE = 32 * V;
    R carry = (R)0;  // A_{t+1} (GAE) or ret_{t+1} (n-step) entering the tile from the right
    for (int hi = ((T + TILE - 1) / TILE) * TILE; hi > 0; hi -= TILE) {
        const int t0 = hi - TILE + lane * V;  // this lane's first step
        float r[V], v[V + 1], d[V], bs[V];
        uint8_t se[V];
        if (V == 4 && VEC && t0 + V <= T) {  // 16-byte loads: T % 4 == 0 and 16-B aligned rows (checked on the host)
            const float4 r4 = *reinterpret_cast<const float4 *>(rew + base + t0);
            const float4 v4 = *reinterpret_cast<const float4 *>(val + base + t0);
            const float4 d4 = *reinterpret_cast<const float4 *>(term + base + t0);
            const uchar4 s4 = *reinterpret_cast<const uchar4 *>(seg_end + base + t0);
            r[0] = r4.x, r[1] = r4.y, r[2] = r4.z, r[3] = r4.w;
            v[0] = v4.x, v[1] = v4.y, v[2] = v4.z, v[3] = v4.w;
            d[0] = d4.x, d[1] = d4.y, d[2] = d4.z, d[3] = d4.w;
            se[0] = s4.x, se[1] = s4.y, se[2] = s4.z, se[3] = s4.w;
            if (s4.x | s4.y | s4.z | s4.w) {
                const float4 b4 = *reinterpret_cast<const float4 *>(boot + base + t0);
                bs[0] = b4.x, bs[1] = b4.y, bs[2] = b4.z, bs[3] = b4.w;
            } else {
                bs[0] = bs[1] = bs[2] = bs[3] = 0.f;
            }
        } else {
#pragma unroll
            for (int j = 0; j < V; ++j) {
                int t = t0 + j;
                bool in = t < T;
                r[j] = in ? rew[base + t] : 0.f;
                v[j] = in ? val[base + t] : 0.f;
                d[j] = in ? term[base + t] : 0.f;
                se[j] = in ? seg_end[base + t] : (uint8_t)1;
                bs[j] = (in && se[j]) ? boot[base + t] : 0.f;
            }
        }
        {
            // V_{t+1} of the lane's last step = the next lane's first value; lane 31 reads it from memory
            float nxt = __shfl_down_sync(0xffffffffu, v[0], 1);
            int t = t0 + V;
            if (lane == 31) nxt = (t < T) ? val[base + t] : 0.f;
            v[V] = nxt;
        }
        // local suffix maps, serial from the lane's last step to its first
        Affine<R> loc[V];
        float tdres[V];  // one-step TD residual for the non-GAE advantage
        Affine<R> acc = {(R)1, (R)0};
#pragma unroll
        for (int j = V - 1; j >= 0; --j) {
            Affine<R> f;
            float vnext = se[j] ? bs[j] : v[j + 1];
            if (GAE) {
                float nd = 1.f - d[j];
                float delta = r[j] + nd * gamma * vnext - v[j];
                f.a = se[j] ? (R)0 : (R)(nd * gl);
                f.b = (R)delta;
            } else {
                // ret_t = r_t + gamma * (seg_end ? bootstrap : ret_{t+1})  in R = double
                f.a = se[j] ? (R)0 : (R)gamma;
                f.b = se[j] ? (R)r[j] + (R)gamma * (R)bs[j] : (R)r[j];
                tdres[j] = r[j] + gamma * vnext - v[j];
            }
            acc = compose(f, acc);
            loc[j] = acc;
        }
        // exclusive scan across lanes from the right: E_l = acc_{l+1} o acc_{l+2} o ... o acc_31
        Affine<R> inc = acc;  // inclusive suffix composition
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            Affine<R> other = {shfl_down_t<R>(inc.a, o), shfl_down_t<R>(inc.b, o)};
            if (lane + o < 32) inc = compose(inc, other);
        }
        Affine<R> excl = {shfl_down_t<R>(inc.a, 1), shfl_down_t<R>(inc.b, 1)};
        if (lane == 31) excl = {(R)1, (R)0};
        const R x_in = excl.a * carry + excl.b;  // value entering this lane from the right
        float a_o[V], r_o[V];
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int t = t0 + j;
            R y = loc[j].a * x_in + loc[j].b;
            float a_out, r_out;
            if (GAE) {
                a_out = (float)y;
                r_out = a_out + v[j];
            } else {
                r_out = (float)y;
                a_out = tdres[j];
            }
            const bool ok = t < cov;
            a_o[j] = ok ? a_out : 0.f;
            r_o[j] = ok ? r_out : 0.f;
        }
        if (V == 4 && VEC && t0 + V <= T) {
            *reinterpret_cast<float4 *>(adv + base + t0) = make_float4(a_o[0], a_o[1], a_o[2], a_o[3]);
            *reinterpret_cast<float4 *>(ret + base + t0) = make_float4(r_o[0], r_o[1], r_o[2], r_o[3]);
        } else {
#pragma unroll
            for (int j = 0; j < V; ++j)
                if (t0 + j < T) {
                    adv[base + t0 + j] = a_o[j];
                    ret[base + t0 + j] = r_o[j];
                }
        }
        // carry for the next (earlier) tile = value at this tile's first step = lane 0's y at j=0
        R first = loc[0].a * x_in + loc[0].b;
        carry = __shfl_sync(0xffffffffu, first, 0);
    }
}

extern "C" int xb_gae_scan(const float *rew, const float *val, const float *term, const uint8_t *seg_end,
                           const float *bootstrap, const int32_t *covered, float *adv, float *ret, int N, int T,
                           float gamma, float lam, int use_gae, void *stream) {
    if (!rew || !val || !term || !seg_end || !bootstrap || !adv || !ret) return XB_EINVAL;
    if (N <= 0 || T <= 0) return XB_EINVAL;
    const int warps_per_block = 4;
    dim3 grid((N + warps_per_block - 1) / warps_per_block), block(32 * warps_per_block);
    cudaStream_t s = (cudaStream_t)stream;
    const bool vec = (T % 4 == 0) && xb_aligned(rew, 16) && xb_aligned(val, 16) && xb_aligned(term, 16) &&
                     xb_aligned(bootstrap, 16) && xb_aligned(adv, 16) && xb_aligned(ret, 16) && xb_aligned(seg_end, 4);
#define XB_GAE(RT, G, VECF) \
    gae_scan_kernel<RT, G, 4, VECF><<<grid, block, 0, s>>>(rew, val, term, seg_end, bootstrap, covered, adv, ret, N, T, gamma, lam)
    if (use_gae) {
        if (vec) XB_GAE(float, true, true); else XB_GAE(float, true, false);
    } else {
        if (vec) XB_GAE(double, false, true); else XB_GAE(double, false, false);
    }
#undef XB_GAE
    return xb_launch_status();
}

// ---- K2 with value normalisation: MARL_OnPolicyBuffer.finish_path (memory_tools_marl.py:208-236)
// Rows are (env, agent) pairs.  Values and the GAE bootstrap are denormalised with the ValueNorm state read here,
// in float32 as ValueNorm.denormalize computes it; the recursion runs in float64 like the reference's Python floats;
// returns are rounded to float32 and advantages = returns - denorm(values) in float32.  Only steps in
// [start[row], covered[row]) are written, so a path keeps the state of the moment it was finished.
__device__ __forceinline__ void vn_state(const float *rm, const float *rmsq, const float *dt, float &mean, float &stdv) {
    mean = 0.f, stdv = 1.f;
    if (!rm) return;
    const float d = fmaxf(dt[0], 1e-5f);
    mean = __fdiv_rn(rm[0], d);
    const float var = fmaxf(__fsub_rn(__fdiv_rn(rmsq[0], d), __fmul_rn(mean, mean)), 1e-2f);
    stdv = __fsqrt_rn(var);
}
__device__ __forceinline__ float vn_denorm(float x, bool on, float mean, float stdv) {
    return on ? __fadd_rn(__fmul_rn(x, stdv), mean) : x;
}

// use_gae: the same warp scan of affine maps as K2 (one warp per row), in float64
__global__ void __launch_bounds__(128) marl_gae_kernel(const float *__restrict__ rew, const float *__restrict__ val,
                                                       const float *__restrict__ term,
                                                       const uint8_t *__restrict__ seg_end,
                                                       const float *__restrict__ boot, const int32_t *__restrict__ start,
                                                       const int32_t *__restrict__ covered, float *__restrict__ adv,
                                                       float *__restrict__ ret, int N, int T, double gamma, double lam,
                                                       const float *rm, const float *rmsq, const float *dt) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= N) return;
    float mean, stdv;
    vn_state(rm, rmsq, dt, mean, stdv);
    const bool on = rm != nullptr;
    const int64_t base = (int64_t)row * T;
    const int beg = start ? start[row] : 0, cov = covered ? covered[row] : T;
    constexpr int V = 4, TILE = 32 * V;
    double carry = 0.0;
    for (int hi = ((T + TILE - 1) / TILE) * TILE; hi > 0; hi -= TILE) {
        const int t0 = hi - TILE + lane * V;
        float v[V + 1];
        Affine<double> loc[V];
        Affine<double> acc = {1.0, 0.0};
#pragma unroll
        for (int j = 0; j < V; ++j) v[j] = (t0 + j < T) ? vn_denorm(val[base + t0 + j], on, mean, stdv) : 0.f;
        {
            float nxt = __shfl_down_sync(0xffffffffu, v[0], 1);
            if (lane == 31) nxt = (t0 + V < T) ? vn_denorm(val[base + t0 + V], on, mean, stdv) : 0.f;
            v[V] = nxt;
        }
#pragma unroll
        for (int j = V - 1; j >= 0; --j) {
            const int t = t0 + j;
            const bool in = t < T;
            const bool se = in ? seg_end[base + t] != 0 : true;
            const double nd = in ? 1.0 - (double)term[base + t] : 1.0;
            const double vnext = (double)((in && se) ? vn_denorm(boot[base + t], on, mean, stdv) : v[j + 1]);
            const double r = in ? (double)rew[base + t] : 0.0;
            Affine<double> f;
            f.a = se ? 0.0 : nd * gamma * lam;
            f.b = r + nd * gamma * vnext - (double)v[j];
            acc = compose(f, acc);
            loc[j] = acc;
        }
        Affine<double> inc = acc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            Affine<double> other = {shfl_down_t<double>(inc.a, o), shfl_down_t<double>(inc.b, o)};
            if (lane + o < 32) inc = compose(inc, other);
        }
        Affine<double> excl = {shfl_down_t<double>(inc.a, 1), shfl_down_t<double>(inc.b, 1)};
        if (lane == 31) excl = {1.0, 0.0};
        const double x_in = excl.a * carry + excl.b;
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const int t = t0 + j;
            if (t < T && t >= beg && t < cov) {
                const float r_out = (float)(loc[j].a * x_in + loc[j].b + (double)v[j]);
                ret[base + t] = r_out;
                adv[base + t] = __fsub_rn(r_out, v[j]);
            }
        }
        const double first = loc[0].a * x_in + loc[0].b;
        carry = __shfl_sync(0xffffffffu, first, 0);
    }
}

// not use_gae: returns_[t] = r_t + (1 - d_t) * gamma * returns_[t+1], stored to float32 at every step as the reference's
// float32 array does (a serial recursion, one thread per row); the bootstrap is the raw stored value, not denormalised
__global__ void __launch_bounds__(128) marl_returns_kernel(const float *__restrict__ rew, const float *__restrict__ val,
                                                           const float *__restrict__ term,
                                                           const uint8_t *__restrict__ seg_end,
                                                           const float *__restrict__ boot,
                                                           const int32_t *__restrict__ start,
                                                           const int32_t *__restrict__ covered, float *__restrict__ adv,
                                                           float *__restrict__ ret, int N, int T, double gamma,
                                                           const float *rm, const float *rmsq, const float *dt) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= N) return;
    float mean, stdv;
    vn_state(rm, rmsq, dt, mean, stdv);
    const bool on = rm != nullptr;
    const int64_t base = (int64_t)row * T;
    const int beg = start ? start[row] : 0, cov = covered ? covered[row] : T;
    float next = 0.f;
    for (int t = cov - 1; t >= beg; --t) {
        if (seg_end[base + t]) next = boot[base + t];
        const double nd = 1.0 - (double)term[base + t];
        next = (float)((double)rew[base + t] + nd * gamma * (double)next);
        ret[base + t] = next;
        adv[base + t] = __fsub_rn(next, vn_denorm(val[base + t], on, mean, stdv));
    }
}

extern "C" int xb_gae_scan_vn(const float *rew, const float *val, const float *term, const uint8_t *seg_end,
                              const float *bootstrap, const int32_t *start, const int32_t *covered, float *adv,
                              float *ret, int N, int T, double gamma, double lam, int use_gae,
                              const float *running_mean, const float *running_mean_sq, const float *debiasing_term,
                              void *stream) {
    if (!rew || !val || !term || !seg_end || !bootstrap || !adv || !ret) return XB_EINVAL;
    if (N <= 0 || T <= 0) return XB_EINVAL;
    const bool some = running_mean || running_mean_sq || debiasing_term;
    if (some && !(running_mean && running_mean_sq && debiasing_term)) return XB_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    if (use_gae) {
        const int warps_per_block = 4;
        marl_gae_kernel<<<(N + warps_per_block - 1) / warps_per_block, 32 * warps_per_block, 0, s>>>(
            rew, val, term, seg_end, bootstrap, start, covered, adv, ret, N, T, gamma, lam, running_mean,
            running_mean_sq, debiasing_term);
    } else {
        marl_returns_kernel<<<(N + 127) / 128, 128, 0, s>>>(rew, val, term, seg_end, bootstrap, start, covered, adv,
                                                             ret, N, T, gamma, running_mean, running_mean_sq,
                                                             debiasing_term);
    }
    return xb_launch_status();
}

// =====================================================================================================
// K3  gathers
// =====================================================================================================
// ---- generic small-row gather (any row_bytes % 4 == 0): one warp per row chunk, 4 B words.
__global__ void __launch_bounds__(256) gather_rows_small_kernel(const uint8_t *__restrict__ src,
                                                                const int64_t *__restrict__ idx, int64_t B,
                                                                int64_t row_bytes, uint8_t *__restrict__ dst) {
    const int64_t words = row_bytes / 4;
    const int64_t total = B * words;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        int64_t b = i / words, w = i - b * words;
        int64_t s = idx ? idx[b] : b;
        reinterpret_cast<uint32_t *>(dst)[i] = *reinterpret_cast<const uint32_t *>(src + s * row_bytes + w * 4);
    }
}

// ---- bulk-async byte gather: one elected thread per CTA drives a ring of shared-memory stages;
//      global->shared and shared->global both run on the TMA unit (UBLKCP), no register traffic at all.
constexpr int GR_STAGES = 4;
constexpr uint32_t GR_CHUNK = 28224;  // bytes per stage (one Atari observation row; generic rows are split)

__global__ void __launch_bounds__(32) gather_rows_bulk_kernel(const uint8_t *__restrict__ src,
                                                              const int64_t *__restrict__ idx, int64_t B,
                                                              int64_t row_bytes, uint8_t *__restrict__ dst,
                                                              uint32_t chunk, int chunks_per_row) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t full[GR_STAGES];
    if (threadIdx.x != 0) return;  // single-thread kernel: the copy engines do the work
    for (int s = 0; s < GR_STAGES; ++s) mbar_init(&full[s], 1);
    mbar_fence_init();
    const int64_t items = B * chunks_per_row;
    // this CTA's items: blockIdx.x, blockIdx.x + gridDim.x, ...
    auto item_ptrs = [&](int64_t it, const uint8_t *&g_src, uint8_t *&g_dst, uint32_t &bytes) {
        int64_t b = it / chunks_per_row;
        int c = (int)(it - b * chunks_per_row);
        int64_t srow = idx ? idx[b] : b;
        int64_t off = (int64_t)c * chunk;
        int64_t rem = row_bytes - off;
        bytes = (uint32_t)(rem < (int64_t)chunk ? rem : chunk);
        g_src = src + srow * row_bytes + off;
        g_dst = dst + b * row_bytes + off;
    };
    int64_t n_mine = items > (int64_t)blockIdx.x ? (items - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    // prologue: fill the ring
    for (int k = 0; k < GR_STAGES && k < n_mine; ++k) {
        const uint8_t *gs;
        uint8_t *gd;
        uint32_t bytes;
        item_ptrs(blockIdx.x + (int64_t)k * gridDim.x, gs, gd, bytes);
        mbar_expect_tx(&full[k], bytes);
        bulk_g2s(smem + (size_t)k * chunk, gs, bytes, &full[k]);
    }
    for (int64_t k = 0; k < n_mine; ++k) {
        int s = (int)(k % GR_STAGES);
        uint32_t parity = (uint32_t)((k / GR_STAGES) & 1);
        const uint8_t *gs;
        uint8_t *gd;
        uint32_t bytes;
        item_ptrs(blockIdx.x + k * gridDim.x, gs, gd, bytes);
        mbar_wait(&full[s], parity);
        fence_proxy_async();
        bulk_s2g(gd, smem + (size_t)s * chunk, bytes);
        bulk_commit();
        // refill the stage used by item k-1 (its store was committed one iteration ago) with item k-1+STAGES
        int64_t kn = k - 1 + GR_STAGES;
        if (k >= 1 && kn < n_mine) {
            bulk_wait_read<1>();  // all but the newest store have finished READING shared memory
            int sn = (int)(kn % GR_STAGES);
            const uint8_t *gs2;
            uint8_t *gd2;
            uint32_t b2;
            item_ptrs(blockIdx.x + kn * gridDim.x, gs2, gd2, b2);
            mbar_expect_tx(&full[sn], b2);
            bulk_g2s(smem + (size_t)sn * chunk, gs2, b2, &full[sn]);
        }
    }
    bulk_wait_all<0>();
}

extern "C" int xb_gather_rows(const void *src, const int64_t *idx, int64_t B, int64_t row_bytes, void *dst,
                              void *stream) {
    if (!src || !dst || B < 0 || row_bytes <= 0) return XB_EINVAL;
    if (B == 0) return XB_OK;
    if (row_bytes & 3) return XB_EALIGN;
    cudaStream_t s = (cudaStream_t)stream;
    const bool bulk = (row_bytes % 16 == 0) && row_bytes >= 2048 && xb_aligned(src, 16) && xb_aligned(dst, 16);
    if (!bulk) {
        if (!xb_aligned(src, 4) || !xb_aligned(dst, 4)) return XB_EALIGN;
        int64_t total = B * (row_bytes / 4);
        int64_t want = (total + 255) / 256, cap = (int64_t)xb_sm_count() * 8;
        gather_rows_small_kernel<<<(int)(want < cap ? want : cap), 256, 0, s>>>((const uint8_t *)src, idx, B, row_bytes,
                                                                              (uint8_t *)dst);
        return xb_launch_status();
    }
    uint32_t chunk = row_bytes <= (int64_t)GR_CHUNK ? (uint32_t)row_bytes : GR_CHUNK;
    int chunks_per_row = (int)((row_bytes + chunk - 1) / chunk);
    size_t smem = (size_t)GR_STAGES * chunk;
    static bool attr_set = false;
    if (!attr_set) {
        cudaFuncSetAttribute(gather_rows_bulk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)(GR_STAGES * GR_CHUNK));
        attr_set = true;
    }
    int64_t items = B * chunks_per_row;
    int64_t ctas = (int64_t)xb_sm_count() * 2;  // 2 x 113 KB rings per SM
    if (ctas > items) ctas = items;
    gather_rows_bulk_kernel<<<(int)ctas, 32, smem, s>>>((const uint8_t *)src, idx, B, row_bytes, (uint8_t *)dst, chunk,
                                                        chunks_per_row);
    return xb_launch_status();
}

// ---- observation gather with fused u8 -> float conversion (u8/255.0 correctly rounded through a LUT).
// Rows are staged into shared memory by the bulk-async engine (one elected thread), all threads then read
// 16 pixels from shared memory, convert, and write 16-byte vectors to global memory.
constexpr int GO_STAGES = 3;
constexpr int GO_THREADS = 256;

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
    __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}
__device__ __forceinline__ uint32_t pack_f16x2(float a, float b) {
    __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<uint32_t *>(&h);
}

template <int FORMAT>
__global__ void __launch_bounds__(GO_THREADS) gather_obs_kernel(const uint8_t *__restrict__ src,
                                                                const int64_t *__restrict__ idx, int64_t B,
                                                                int row_bytes, int H, int W, void *__restrict__ dstv) {
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ __align__(8) uint64_t full[GO_STAGES];
    __shared__ float lut[256];
    const int tid = threadIdx.x;
    lut[tid & 255] = __fdiv_rn((float)(tid & 255), 255.0f);
    if (tid == 0) {
        for (int s = 0; s < GO_STAGES; ++s) mbar_init(&full[s], 1);
        mbar_fence_init();
    }
    __syncthreads();
    const int64_t n_mine = B > (int64_t)blockIdx.x ? (B - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    auto issue = [&](int64_t k) {
        int s = (int)(k % GO_STAGES);
        int64_t b = blockIdx.x + k * gridDim.x;
        int64_t srow = idx ? idx[b] : b;
        mbar_expect_tx(&full[s], (uint32_t)row_bytes);
        bulk_g2s(smem + (size_t)s * row_bytes, src + srow * (int64_t)row_bytes, (uint32_t)row_bytes, &full[s]);
    };
    if (tid == 0)
        for (int k = 0; k < GO_STAGES - 1 && k < n_mine; ++k) issue(k);
    // bytes of the u8 row consumed per thread-iteration: chosen so that ONE store instruction of a warp covers
    // 512 contiguous bytes (fully coalesced 16 B per lane); NCHW needs a 4-pixel x 4-channel block per thread.
    constexpr int IN_BYTES = (FORMAT == XB_OBS_F32_NHWC) ? 4 : (FORMAT == XB_OBS_F32_NCHW ? 16 : 8);
    const int units = row_bytes / IN_BYTES;
    for (int64_t k = 0; k < n_mine; ++k) {
        const int s = (int)(k % GO_STAGES);
        const uint32_t parity = (uint32_t)((k / GO_STAGES) & 1);
        // stage (k-1)%STAGES was fully consumed before the __syncthreads at the end of iteration k-1
        if (tid == 0 && k + GO_STAGES - 1 < n_mine) issue(k + GO_STAGES - 1);
        mbar_wait(&full[s], parity);
        const uint8_t *row = smem + (size_t)s * row_bytes;
        const int64_t b = blockIdx.x + k * gridDim.x;
#pragma unroll 4
        for (int c = tid; c < units; c += GO_THREADS) {
            if (FORMAT == XB_OBS_F32_NHWC) {
                const uint32_t w = *reinterpret_cast<const uint32_t *>(row + c * 4);
                uint4 o = {__float_as_uint(lut[w & 0xffu]), __float_as_uint(lut[(w >> 8) & 0xffu]),
                           __float_as_uint(lut[(w >> 16) & 0xffu]), __float_as_uint(lut[w >> 24])};
                stg_stream16(reinterpret_cast<float *>(dstv) + b * (int64_t)row_bytes + (int64_t)c * 4, o);
            } else if (FORMAT == XB_OBS_F32_NCHW) {
                // 16 bytes = 4 pixels (w..w+3) x 4 channels; plane ch gets a float4 of the 4 pixels
                const uint4 p = *reinterpret_cast<const uint4 *>(row + c * 16);
                const uint32_t w[4] = {p.x, p.y, p.z, p.w};
                const int pix = c * 4;  // pixel index within the image (h*W + w), W % 4 == 0
                float *out = reinterpret_cast<float *>(dstv) + b * (int64_t)row_bytes;
                const int64_t plane = (int64_t)H * W;
#pragma unroll
                for (int ch = 0; ch < 4; ++ch) {
                    uint4 o = {__float_as_uint(lut[(w[0] >> (8 * ch)) & 0xffu]),
                               __float_as_uint(lut[(w[1] >> (8 * ch)) & 0xffu]),
                               __float_as_uint(lut[(w[2] >> (8 * ch)) & 0xffu]),
                               __float_as_uint(lut[(w[3] >> (8 * ch)) & 0xffu])};
                    stg_stream16(out + ch * plane + pix, o);
                }
            } else {
                const uint2 p = *reinterpret_cast<const uint2 *>(row + c * 8);
                float f[8];
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    f[j] = lut[(p.x >> (8 * j)) & 0xffu];
                    f[4 + j] = lut[(p.y >> (8 * j)) & 0xffu];
                }
                uint4 o;
                if (FORMAT == XB_OBS_BF16_NHWC)
                    o = {pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]),
                         pack_bf16x2(f[6], f[7])};
                else
                    o = {pack_f16x2(f[0], f[1]), pack_f16x2(f[2], f[3]), pack_f16x2(f[4], f[5]),
                         pack_f16x2(f[6], f[7])};
                stg_stream16(reinterpret_cast<uint16_t *>(dstv) + b * (int64_t)row_bytes + (int64_t)c * 8, o);
            }
        }
        __syncthreads();  // every thread is done with stage s before it is refilled
    }
}

extern "C" int xb_gather_obs(const uint8_t *src, const int64_t *idx, int64_t B, int H, int W, int C, void *dst,
                             int format, void *stream) {
    if (!src || !dst || B < 0 || H <= 0 || W <= 0 || C <= 0) return XB_EINVAL;
    if (B == 0) return XB_OK;
    const int64_t row_bytes = (int64_t)H * W * C;
    if (format == XB_OBS_U8) return xb_gather_rows(src, idx, B, row_bytes, dst, stream);
    if (row_bytes % 16 != 0 || !xb_aligned(src, 16) || !xb_aligned(dst, 16)) return XB_EALIGN;
    if (row_bytes * GO_STAGES > 200 * 1024) return XB_ERANGE;
    if (format == XB_OBS_F32_NCHW && (C != 4 || (W & 3))) return XB_ERANGE;
    cudaStream_t s = (cudaStream_t)stream;
    size_t smem = (size_t)GO_STAGES * row_bytes;
    int64_t ctas = (int64_t)xb_sm_count() * 2;
    if (ctas > B) ctas = B;
#define XB_LAUNCH_GO(FMT)                                                                                         \
    do {                                                                                                          \
        static bool set_##FMT = false;                                                                            \
        if (!set_##FMT) {                                                                                         \
            cudaFuncSetAttribute(gather_obs_kernel<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); \
            set_##FMT = true;                                                                                     \
        }                                                                                                         \
        gather_obs_kernel<FMT><<<(int)ctas, GO_THREADS, smem, s>>>(src, idx, B, (int)row_bytes, H, W, dst);       \
    } while (0)
    switch (format) {
        case XB_OBS_F32_NHWC: XB_LAUNCH_GO(XB_OBS_F32_NHWC); break;
        case XB_OBS_F32_NCHW: XB_LAUNCH_GO(XB_OBS_F32_NCHW); break;
        case XB_OBS_BF16_NHWC: XB_LAUNCH_GO(XB_OBS_BF16_NHWC); break;
        case XB_OBS_F16_NHWC: XB_LAUNCH_GO(XB_OBS_F16_NHWC); break;
        default: return XB_EINVAL;
    }
#undef XB_LAUNCH_GO
    return xb_launch_status();
}

// ---- scalar-field gather + per-minibatch advantage normalisation --------------------------------------
__global__ void __launch_bounds__(256) gather_scalars_kernel(const float *__restrict__ fields, int64_t slots,
                                                             const int64_t *__restrict__ idx, int64_t B, int F,
                                                             float *__restrict__ out, int adv_field,
                                                             float *__restrict__ stats, double *__restrict__ scratch) {
    __shared__ double red[2 * 32];
    double acc[2] = {0.0, 0.0};
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x) {
        const int64_t s = idx ? idx[b] : b;
        for (int f = 0; f < F; ++f) {
            float x = fields[(int64_t)f * slots + s];
            out[(int64_t)f * B + b] = x;
            if (f == adv_field) {
                acc[0] += (double)x;
                acc[1] += (double)x * (double)x;
            }
        }
    }
    if (adv_field < 0) return;
    grid_sum_finalize<2>(acc, scratch, red, [&](double(&tot)[2]) {
        double mean = tot[0] / (double)B;
        double var = tot[1] / (double)B - mean * mean;
        if (var < 0.0) var = 0.0;
        stats[0] = (float)mean;
        stats[1] = (float)sqrt(var);
    });
}

__global__ void __launch_bounds__(256) adv_normalize_kernel(float *__restrict__ adv, int64_t B,
                                                            const float *__restrict__ stats) {
    const float mean = stats[0];
    const float denom = __fadd_rn(stats[1], 1e-8f);
    for (int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += (int64_t)gridDim.x * blockDim.x)
        adv[b] = __fdiv_rn(__fsub_rn(adv[b], mean), denom);
}

extern "C" int64_t xb_scratch_doubles(void) { return XB_SCRATCH_DOUBLES; }

// normalise with GIVEN statistics (sharded minibatches: the global mean / std of the minibatch come from one all-reduce
// per epoch, memory_tools.global_adv_stats)
extern "C" int xb_adv_normalize(float *adv, int64_t B, const float *stats, void *stream) {
    if (!adv || !stats || B <= 0) return XB_EINVAL;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    adv_normalize_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(adv, B, stats);
    return xb_launch_status();
}

extern "C" int xb_gather_scalars(const float *fields, int64_t slots, const int64_t *idx, int64_t B, int F, float *out,
                                 int adv_field, float *stats_out, double *scratch, void *stream) {
    if (!fields || !out || B <= 0 || F <= 0 || slots <= 0 || adv_field >= F) return XB_EINVAL;
    if (adv_field >= 0 && (!stats_out || !scratch)) return XB_EINVAL;
    cudaStream_t s = (cudaStream_t)stream;
    int64_t want = (B + 255) / 256;
    int grid = (int)(want < XB_MAX_PARTIALS ? want : XB_MAX_PARTIALS);
    gather_scalars_kernel<<<grid, 256, 0, s>>>(fields, slots, idx, B, F, out, adv_field, stats_out, scratch);
    int st = xb_launch_status();
    if (st != XB_OK || adv_field < 0) return st;
    adv_normalize_kernel<<<grid, 256, 0, s>>>(out + (int64_t)adv_field * B, B, stats_out);
    return xb_launch_status();
}
