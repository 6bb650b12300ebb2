// wf_fft.cuh — register-resident DFT building blocks for the sm_90a STFT kernels.
//
// A thread holds R complex points in registers (R = 2..32) and performs a radix-2 decimation-in-
// frequency network on them with compile-time twiddles; the result of bin k ends up in register
// bitrev(k), which callers absorb into their (compile-time) store indices, so no data movement is
// spent on reordering.  These are the "warp-shuffle / register butterflies" of the design: all
// inter-thread exchange happens once per Stockham pass through padded shared memory.
//
// Replaces (together with wf_kernels.cuh) the FFTW codelets the reference executes through
// fftwf_execute (src/source_generic.cpp:106; deps/fftw-3.3.11/rdft/ct-hc2c.c:59-70).
#pragma once
#include <cuda_runtime.h>

namespace wf {

// ---- compile-time sin/cos (double precision Taylor with octant reduction) -------------------------
namespace cx {
constexpr double kPi = 3.14159265358979323846264338327950288;
constexpr double sin_taylor(double x)
{ // |x| <= pi/4
    double x2 = x * x, term = x, sum = x;
    for(int n = 1; n < 12; ++n)
    {
        term *= -x2 / ((2.0 * n) * (2.0 * n + 1.0));
        sum += term;
    }
    return sum;
}
constexpr double cos_taylor(double x)
{ // |x| <= pi/4
    double x2 = x * x, term = 1.0, sum = 1.0;
    for(int n = 1; n < 12; ++n)
    {
        term *= -x2 / ((2.0 * n - 1.0) * (2.0 * n));
        sum += term;
    }
    return sum;
}
// cos(2 pi k / n), sin(2 pi k / n) for 0 <= k < n, exact symmetry handling by octant
constexpr double cos2pi(int k, int n)
{
    k %= n;
    if(8 * k <= n) return cos_taylor(2.0 * kPi * k / n);
    if(8 * k <= 3 * n) return -sin_taylor(2.0 * kPi * k / n - kPi / 2);
    if(8 * k <= 5 * n) return -cos_taylor(2.0 * kPi * k / n - kPi);
    if(8 * k <= 7 * n) return sin_taylor(2.0 * kPi * k / n - 3 * kPi / 2);
    return cos_taylor(2.0 * kPi * k / n - 2 * kPi);
}
constexpr double sin2pi(int k, int n)
{
    k %= n;
    if(8 * k <= n) return sin_taylor(2.0 * kPi * k / n);
    if(8 * k <= 3 * n) return cos_taylor(2.0 * kPi * k / n - kPi / 2);
    if(8 * k <= 5 * n) return -sin_taylor(2.0 * kPi * k / n - kPi);
    if(8 * k <= 7 * n) return -cos_taylor(2.0 * kPi * k / n - 3 * kPi / 2);
    return sin_taylor(2.0 * kPi * k / n - 2 * kPi);
}
} // namespace cx

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 w)
{
    return make_float2(fmaf(a.x, w.x, -a.y * w.y), fmaf(a.x, w.y, a.y * w.x));
}

// multiply by the compile-time twiddle W_L^J = exp(-2 pi i J / L)
template<int J, int L>
__device__ __forceinline__ float2 mul_tw(float2 a)
{
    if constexpr(J == 0)
        return a;
    else if constexpr(4 * J == L) // -i
        return make_float2(a.y, -a.x);
    else if constexpr(8 * J == L) // (1 - i)/sqrt2
    {
        constexpr float h = 0.70710678118654752440f;
        return make_float2((a.x + a.y) * h, (a.y - a.x) * h);
    }
    else if constexpr(8 * J == 3 * L) // (-1 - i)/sqrt2
    {
        constexpr float h = 0.70710678118654752440f;
        return make_float2((a.y - a.x) * h, -(a.x + a.y) * h);
    }
    else
    {
        constexpr float c = (float)cx::cos2pi(J, L);
        constexpr float s = -(float)cx::sin2pi(J, L);
        return make_float2(fmaf(a.x, c, -a.y * s), fmaf(a.x, s, a.y * c));
    }
}

template<int R>
__host__ __device__ constexpr int bitrev(int k)
{
    int r = 0;
    for(int b = 1; b < R; b <<= 1)
    {
        r = (r << 1) | (k & 1);
        k >>= 1;
    }
    return r;
}

// One DIF stage on the sub-block [BASE, BASE+L): v[b+j] = a+c, v[b+j+L/2] = (a-c) W_L^j
template<int L, int BASE, int J, typename V>
__device__ __forceinline__ void dif_bfly(V &v)
{
    if constexpr(J < L / 2)
    {
        const float2 a = v[BASE + J];
        const float2 c = v[BASE + J + L / 2];
        v[BASE + J] = cadd(a, c);
        v[BASE + J + L / 2] = mul_tw<J, L>(csub(a, c));
        dif_bfly<L, BASE, J + 1>(v);
    }
}

template<int L, int BASE, typename V>
__device__ __forceinline__ void dif_block(V &v)
{
    if constexpr(L >= 2)
    {
        dif_bfly<L, BASE, 0>(v);
        dif_block<L / 2, BASE>(v);
        dif_block<L / 2, BASE + L / 2>(v);
    }
}

// In-place forward DFT of v[0..R): afterwards X[k] == v[bitrev<R>(k)].
template<int R>
__device__ __forceinline__ void dft_bitrev(float2 (&v)[R])
{
    dif_block<R, 0>(v);
}

} // namespace wf

// ---------------------------------------------------------------------------------------------------
// Complex arithmetic on a 64-bit register pair (re = low half, im = high half).  Hopper has no packed FP32
// datapath, so every elementwise operation is two scalar IEEE round-to-nearest operations; the explicit
// __fadd_rn / __fmul_rn / __fmaf_rn forms keep ptxas from contracting a separate mul + add into one FMA, so
// each lane rounds exactly as written.  The pair packing (mov.b64) is a register renaming and costs nothing.
// ---------------------------------------------------------------------------------------------------
namespace wf {
namespace pk {

typedef unsigned long long c64;

__device__ __forceinline__ c64 make(float re, float im)
{
    c64 r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(re), "f"(im));
    return r;
}
__device__ __forceinline__ void split(c64 a, float &re, float &im)
{
    asm("mov.b64 {%0, %1}, %2;" : "=f"(re), "=f"(im) : "l"(a));
}
__device__ __forceinline__ float re(c64 a)
{
    float x, y;
    split(a, x, y);
    return x;
}
__device__ __forceinline__ float im(c64 a)
{
    float x, y;
    split(a, x, y);
    return y;
}
__device__ __forceinline__ c64 from(float2 a) { return make(a.x, a.y); }
__device__ __forceinline__ float2 to_float2(c64 a)
{
    float2 r;
    split(a, r.x, r.y);
    return r;
}
__device__ __forceinline__ c64 add(c64 a, c64 b)
{
    float ax, ay, bx, by;
    split(a, ax, ay);
    split(b, bx, by);
    return make(__fadd_rn(ax, bx), __fadd_rn(ay, by));
}
__device__ __forceinline__ c64 sub(c64 a, c64 b)
{
    float ax, ay, bx, by;
    split(a, ax, ay);
    split(b, bx, by);
    return make(__fsub_rn(ax, bx), __fsub_rn(ay, by));
}
__device__ __forceinline__ c64 mul(c64 a, c64 b) // elementwise
{
    float ax, ay, bx, by;
    split(a, ax, ay);
    split(b, bx, by);
    return make(__fmul_rn(ax, bx), __fmul_rn(ay, by));
}
__device__ __forceinline__ c64 fma(c64 a, c64 b, c64 c) // elementwise a*b+c
{
    float ax, ay, bx, by, cr, ci;
    split(a, ax, ay);
    split(b, bx, by);
    split(c, cr, ci);
    return make(__fmaf_rn(ax, bx, cr), __fmaf_rn(ay, by, ci));
}
__device__ __forceinline__ c64 swap(c64 a)
{
    float x, y;
    split(a, x, y);
    return make(y, x);
}
__device__ __forceinline__ c64 conj(c64 a)
{
    float x, y;
    split(a, x, y);
    return make(x, -y);
}
__device__ __forceinline__ c64 mul_neg_i(c64 a) // a * (-i) = (im, -re)
{
    float x, y;
    split(a, x, y);
    return make(y, -x);
}
// complex multiply by a run-time twiddle w = (c, s):  a*(c,c) + (-a.im, a.re)*(s,s).
__device__ __forceinline__ c64 cmul(c64 a, c64 w)
{
    float x, y, c, s;
    split(a, x, y);
    split(w, c, s);
    return fma(make(-y, x), make(s, s), mul(a, make(c, c)));
}

// multiply by the compile-time twiddle W_L^J = exp(-2 pi i J / L)
template<int J, int L>
__device__ __forceinline__ c64 mul_tw(c64 a)
{
    if constexpr(J == 0)
        return a;
    else if constexpr(4 * J == L)
        return mul_neg_i(a);
    else
    {
        constexpr float c = (float)cx::cos2pi(J, L);
        constexpr float s = -(float)cx::sin2pi(J, L);
        return fma(swap(a), make(-s, s), mul(a, make(c, c)));
    }
}

template<int L, int BASE, int J, int R>
__device__ __forceinline__ void dif_bfly(c64 (&v)[R])
{
    if constexpr(J < L / 2)
    {
        const c64 a = v[BASE + J];
        const c64 c = v[BASE + J + L / 2];
        v[BASE + J] = add(a, c);
        v[BASE + J + L / 2] = mul_tw<J, L>(sub(a, c));
        dif_bfly<L, BASE, J + 1, R>(v);
    }
}
template<int L, int BASE, int R>
__device__ __forceinline__ void dif_block(c64 (&v)[R])
{
    if constexpr(L >= 2)
    {
        dif_bfly<L, BASE, 0, R>(v);
        dif_block<L / 2, BASE, R>(v);
        dif_block<L / 2, BASE + L / 2, R>(v);
    }
}
// In-place forward DFT of v[0..R): afterwards X[k] == v[bitrev<R>(k)].
template<int R>
__device__ __forceinline__ void dft_bitrev(c64 (&v)[R])
{
    dif_block<R, 0, R>(v);
}


// ---- mixed-radix register DFT of any length R <= 32 (compile-time plan) ---------------------------------------------
// Decimation in frequency by the smallest prime factor r of R (R = r*m): for every j < m a radix-r butterfly on
// v[j + m*i], i < r, its output t multiplied by W_R^(j*t) and stored at v[t*m + j]; then the r blocks of length m
// recursively.  Afterwards X[k] == v[perm_mixed(R, k)], perm_mixed(R, k) = (k % r)*m + perm_mixed(m, k / r)
// (for powers of two this is the bit reversal of dft_bitrev).  Radix 2 is add/sub; an odd prime p uses the symmetric form
//   X_k, X_(p-k) = (a0 + sum_j cos(2 pi jk/p)(a_j + a_(p-j)))  -/+  i (sum_j sin(2 pi jk/p)(a_j - a_(p-j)))
// with compile-time constants: (p-1)^2/2 packed FMAs — radix 3, 5, 7, 11, 13 from one template.  These are the "register
// butterflies for radix 3/5" the plugin's non-power-of-two sizes need (800 = 2^5 5^2, 1920 = 2^7 3 5, ...).
constexpr int smallest_factor(int n)
{
    for(int f = 2; f * f <= n; ++f)
        if(n % f == 0)
            return f;
    return n;
}
constexpr int perm_mixed(int R, int k)
{
    if(R <= 1)
        return 0;
    const int r = smallest_factor(R), m = R / r;
    return (k % r) * m + perm_mixed(m, k / r);
}

__device__ __forceinline__ c64 mul_pos_i(c64 a) // a * (+i) = (-im, re)
{
    float x, y;
    split(a, x, y);
    return make(-y, x);
}
__device__ __forceinline__ c64 neg(c64 a)
{
    float x, y;
    split(a, x, y);
    return make(-x, -y);
}
// multiply by W_L^J for any 0 <= J < L (more special cases than mul_tw: -1 and +i)
template<int J, int L>
__device__ __forceinline__ c64 mul_tw_any(c64 a)
{
    if constexpr(J % L == 0)
        return a;
    else if constexpr(2 * (J % L) == L)
        return neg(a);
    else if constexpr(4 * (J % L) == L)
        return mul_neg_i(a);
    else if constexpr(4 * (J % L) == 3 * L)
        return mul_pos_i(a);
    else
    {
        constexpr float c = (float)cx::cos2pi(J % L, L);
        constexpr float s = -(float)cx::sin2pi(J % L, L);
        return fma(swap(a), make(-s, s), mul(a, make(c, c)));
    }
}

// radix-P butterfly (P an odd prime) on a[0..P): a[t] = sum_i a[i] W_P^(i t)
template<int P, int K, int J>
__device__ __forceinline__ void prime_acc(const c64 (&s)[P], const c64 (&d)[P], c64 &m, c64 &n)
{
    if constexpr(J <= (P - 1) / 2)
    {
        constexpr float c = (float)cx::cos2pi((J * K) % P, P);
        constexpr float sn = (float)cx::sin2pi((J * K) % P, P);
        m = fma(s[J], make(c, c), m);
        n = (J == 1) ? mul(d[J], make(sn, sn)) : fma(d[J], make(sn, sn), n);
        prime_acc<P, K, J + 1>(s, d, m, n);
    }
}
template<int P, int K>
__device__ __forceinline__ void prime_out(const c64 a0, const c64 (&s)[P], const c64 (&d)[P], c64 (&out)[P])
{
    if constexpr(K <= (P - 1) / 2)
    {
        c64 m = a0, n = 0ull;
        prime_acc<P, K, 1>(s, d, m, n);
        const c64 in = mul_neg_i(n); // -i n
        out[K] = add(m, in);
        out[P - K] = sub(m, in);
        prime_out<P, K + 1>(a0, s, d, out);
    }
}
template<int P>
__device__ __forceinline__ void bfly_prime(c64 (&a)[P])
{
    c64 s[P], d[P], out[P];
    c64 x0 = a[0];
#pragma unroll
    for(int j = 1; j <= (P - 1) / 2; ++j)
    {
        s[j] = add(a[j], a[P - j]);
        d[j] = sub(a[j], a[P - j]);
        x0 = add(x0, s[j]);
    }
    prime_out<P, 1>(a[0], s, d, out);
    a[0] = x0;
#pragma unroll
    for(int k = 1; k < P; ++k)
        a[k] = out[k];
}

template<int R, int BASE, int RMAX>
__device__ __forceinline__ void dif_mixed(c64 (&v)[RMAX]);

// one DIF step of the block [BASE, BASE + r*m): butterflies j = J .. m-1
template<int r, int m, int BASE, int J, int T, int RMAX>
__device__ __forceinline__ void dif_twiddle(c64 (&v)[RMAX])
{
    if constexpr(T < r)
    {
        v[BASE + T * m + J] = mul_tw_any<J * T, r * m>(v[BASE + T * m + J]);
        dif_twiddle<r, m, BASE, J, T + 1, RMAX>(v);
    }
}
template<int r, int m, int BASE, int J, int RMAX>
__device__ __forceinline__ void dif_step(c64 (&v)[RMAX])
{
    if constexpr(J < m)
    {
        if constexpr(r == 2)
        {
            const c64 a = v[BASE + J], c = v[BASE + J + m];
            v[BASE + J] = add(a, c);
            v[BASE + J + m] = mul_tw_any<J, 2 * m>(sub(a, c));
        }
        else
        {
            c64 a[r];
#pragma unroll
            for(int i = 0; i < r; ++i)
                a[i] = v[BASE + J + m * i];
            bfly_prime<r>(a);
#pragma unroll
            for(int t = 0; t < r; ++t)
                v[BASE + t * m + J] = a[t];
            dif_twiddle<r, m, BASE, J, 1, RMAX>(v);
        }
        dif_step<r, m, BASE, J + 1, RMAX>(v);
    }
}
template<int r, int m, int BASE, int T, int RMAX>
__device__ __forceinline__ void dif_children(c64 (&v)[RMAX])
{
    if constexpr(T < r)
    {
        dif_mixed<m, BASE + T * m, RMAX>(v);
        dif_children<r, m, BASE, T + 1, RMAX>(v);
    }
}
template<int R, int BASE, int RMAX>
__device__ __forceinline__ void dif_mixed(c64 (&v)[RMAX])
{
    if constexpr(R >= 2)
    {
        constexpr int r = smallest_factor(R), m = R / r;
        dif_step<r, m, BASE, 0, RMAX>(v);
        if constexpr(m >= 2)
            dif_children<r, m, BASE, 0, RMAX>(v);
    }
}
// In-place forward DFT of v[0..R) (R <= RMAX): afterwards X[k] == v[perm_mixed(R, k)].
template<int R, int RMAX>
__device__ __forceinline__ void dft_mixed(c64 (&v)[RMAX])
{
    dif_mixed<R, 0, RMAX>(v);
}

} // namespace pk
} // namespace wf
