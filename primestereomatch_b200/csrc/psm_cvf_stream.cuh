// psm_cvf_stream.cuh -- K3: the fused streaming guided-image-filter kernel (the graded kernel).
//
// q = GuidedFilter_cv(I, p) (/root/reference/src/CVF.cpp:72-165) for every owned slice of both cost
// volumes in ONE pass over HBM: p is read once and q written once per voxel; the two chained 8x8
// box stages, a, b, all products and all means stay on the SM.  The reference runs ~90 Mat-sized
// passes per slice for the same result (SURVEY.md section 8a, row a9).
//
// Numerics
//   * cv::boxFilter on CV_32F accumulates in double with running sums along whole rows and columns.
//     Box sums here are fp64 running column sums per row segment (+ newest row, - oldest row) and
//     8-wide row sums, scaled and rounded once to float: OpenCV's float while the fp64 sums are
//     exact.  Outside that domain psm_cvf_ref.cuh filters the slice again in OpenCV's order.
//   * every fp32 operation of a, b and q is a separate IEEE round-to-nearest op in the reference's
//     order (CVF.cpp:87-163): __fmul_rn / __fadd_rn / __fsub_rn, which ptxas never contracts.
//   * PSM_CVF_EXACT: all eight box sums in fp64 -> q bit-exact.
//     PSM_CVF_MIXED: the four stage-1 sums in fp64 (a, b stay bit-exact), the four stage-2 sums
//     (box of a0,a1,a2,b) in fp32 with a FIXED summation tree (below) -> q within ~3e-6 of exact,
//     deterministic and position-independent (tests/mixed_model.py restates it on the CPU).
//
// f32 -> f64 without the conversion (XU) pipe.  F2F has a fraction of the FMA pipe's rate and the exact
// filter needs 24 conversions per voxel, so it binds when every widening uses it.  For a NON-NEGATIVE
// finite float with bit pattern u (zero and denormals included) the 64-bit integer u * 2^29, read
// as a double, is exactly f * 2^-896: the 8-bit exponent field lands in the low bits of the 11-bit
// field (bias error -896), the mantissa lines up, denormals stay denormals of the same scaled
// value, zero stays zero.  That is ONE IMAD.WIDE.U32 on the FMA pipe.  All fp64 sums are kept in
// this 2^-896-scaled domain (a power-of-two scaling commutes with every rounding; nothing
// underflows because the scaled values are multiples of 2^-1045 >= the fp64 denormal quantum) and
// the scale is folded into the constant of the final multiply (2^890 instead of 2^-6).  Signed
// values cost three integer instructions (shift the sign out, IMAD.WIDE, LOP3 the sign back in).
// Rows whose p holds a negative, -0, inf or nan value (a warp vote per row) take a slow path that
// converts with F2F and rescales, and from then on the warp also widens a,b with F2F, so
// non-finite data propagates exactly like in the reference.
//
// Work decomposition (nothing like the reference's per-slice Mat pipeline):
//   warp   = one strip of 128 input columns (112 output columns) of ONE disparity slice, one row segment
//   lane   = 4 consecutive columns -> every global access is a 128-bit load/store
//   CTA    = wpc warps = wpc consecutive slices of the same strip and segment (guide rows hit in L1)
//   stage 1: S1[4 boxes][4 cols] fp64 running column sums of p, I0*p, I1*p, I2*p;
//            row sums = per-lane prefix/suffix sums + 4 fp64 shuffles per box (lane+1 total, lane+2 prefixes)
//   a,b    : CVF.cpp:92-155 with the d-independent adjugate / 1/det precomputed per pixel (K2)
//   ring   : thread-private 8-slot history (512 B per thread) in shared memory, the only on-chip history: stage-1
//            "oldest rows" are re-read from the raw volume (L1/L2).
//            EXACT: slots hold a,b rows;  MIXED: slots hold PAIR rows  pair(t) = ab(t-1) + ab(t)
//   stage 2 EXACT: S2[4 planes][4 cols] fp64 running column sums of a0,a1,a2,b (newest from
//            registers, oldest from the ring); row sums as in stage 1
//   stage 2 MIXED: V(y) = (P(y-3) + P(y-1)) + (P(y+1) + P(y+3)), P(s) = X[r(s-1)] + X[r(s)] with
//            reflected rows, i.e. the tree ((x0+x1)+(x2+x3))+((x4+x5)+(x6+x7)) over window rows
//            y-4..y+3; row sums by the same prefix/suffix scheme in fp32 over ALIGNED 4-column
//            groups (strip origins are multiples of 4, so the tree depends on x only)
//   q = box(b) + sum_c box(a_c) * I_c   (CVF.cpp:157-163)
//
// Column bookkeeping of strip s (X0 = first output column, 112*s; without the packed remainder the
// last strip is shifted left to end at the image edge), lane l (packed remainder: lane within its group):
//   input  columns X0-8+4l .. +3   (p, I)                  halo columns come from the mirrored halo
//   a,b    columns X0-4+4l .. +3   (valid for l <= 29)     of the padded layout (psm_kernels.cuh)
//   output columns X0  +4l .. +3   (valid for l <= 27)
// a,b at columns outside [0,W) must be the REFLECTED a,b (cv::boxFilter reflects its input, which
// for the second stage is a,b) -- not what stage 1 computes there from mirrored p (the 8-wide window
// is asymmetric) -- so border strips overwrite those entries by lane shuffles.
// Packed remainder.  W is rarely a multiple of 112 (1920 = 17 x 112 + 16): a whole warp for the last 16 columns of every
// slice is 1/18 of the kernel's work.  When the remainder needs at most 16 lanes (its columns + 16 halo columns), the
// regular strips stop at 112 * floor(W / 112) and extra "packed" CTAs filter the remainder of 4 (8-lane groups) or 2
// (16-lane groups) SLICES per warp: lane -> (slice group, lane in group), everything below is per lane anyway (base
// pointers, ring, running sums); the shuffles still run over the whole warp and what crosses a group boundary lands in
// the group's halo lanes, whose results are never stored -- exactly like the first and last lanes of a full strip.
// Rows: the top of the image uses weights 1,2,2,2,1 for the first window, the bottom feeds three
// virtual rows from the ring; input rows reflect by index.  These special cases live in
// generic_step; the bulk of the rows run the steady step, which has no data-dependent control
// flow except the warp-uniform fast/slow widening choice.
#pragma once
#include <type_traits>

#include "psm_kernels.cuh"

namespace psm {

constexpr int kStripOut = 112;  // output columns per warp
constexpr int kStripIn = 128;   // input columns per warp
constexpr int kCvfThreads = 96;       // CTA size when the slice count is not a multiple of 4: 3 slice-warps, 4 CTAs/SM (else 128 x 3)
constexpr int kCvfMaxThreads = 448;   // 14 warps: 448 rings of 512 B = 224 KB, the most shared memory one CTA may have (227 KB)

// stage-2 modes (template parameter S2M)
constexpr int kS2Exact = 0;  // fp64 running sums
constexpr int kS2Mixed = 1;  // fp32 pair tree (PSM_CVF_MIXED)

struct CvfParams {
    const float* vol_in[2];   // raw volumes  [Dloc][H][Wp]   (pointer to row 0, column 0)
    float* vol_out[2];        // filtered volumes
    const float* guide[2];    // guide planes [kGuidePlanes][H][Wp]
    const int* guide_flags;   // [2] per view: != 0 when the guide holds negative / non-finite values
    int W, H, Wp, Dloc;
    int nstrips, nseg, seg_rows, ndgroups;
    int remap_sms, remap_ctas;  // SM count and resident CTAs per SM for the block->work remap (0: identity)
    // packed remainder strips (0 = off): blocks >= pack_first filter the W - nstrips*112 rightmost columns with
    // 32 / pack_gl slices per warp (pack_gl = 8 or 16 lanes per slice); see "Packed remainder" in the header comment
    int pack_gl, pack_first, pack_ndg, pack_x0;
    float one, mone;            // +1.0f / -1.0f, passed at run time so that the compiler cannot fold them (exact adds as fma, PA)
};

struct f2x2 { float2 lo, hi; };  // four columns as two pairs
__device__ __forceinline__ f2x2 from4(const float4& v) { return {make_float2(v.x, v.y), make_float2(v.z, v.w)}; }
__device__ __forceinline__ float4 to4(const f2x2& v) { return make_float4(v.lo.x, v.lo.y, v.hi.x, v.hi.y); }
__device__ __forceinline__ f2x2 mul2(const f2x2& a, const f2x2& b)
{
    return {make_float2(__fmul_rn(a.lo.x, b.lo.x), __fmul_rn(a.lo.y, b.lo.y)), make_float2(__fmul_rn(a.hi.x, b.hi.x), __fmul_rn(a.hi.y, b.hi.y))};
}
__device__ __forceinline__ f2x2 add2(const f2x2& a, const f2x2& b)
{
    return {make_float2(fadd(a.lo.x, b.lo.x), fadd(a.lo.y, b.lo.y)), make_float2(fadd(a.hi.x, b.hi.x), fadd(a.hi.y, b.hi.y))};
}
__device__ __forceinline__ f2x2 sub2(const f2x2& a, const f2x2& b)
{
    return {make_float2(fsub(a.lo.x, b.lo.x), fsub(a.lo.y, b.lo.y)), make_float2(fsub(a.hi.x, b.hi.x), fsub(a.hi.y, b.hi.y))};
}
// EXACT add / subtract as an fma: x + y == fma(x, 1, y) and x - y == fma(y, -1, x) with one rounding each; the
// multiplier is a RUN-TIME 1.0f / -1.0f, so ptxas can neither fold nor re-associate it (PA builds).
__device__ __forceinline__ float2 fma2(const float2& a, const float2& b, const float2& c)
{
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// add of operands that are not products
__device__ __forceinline__ f2x2 addp(const f2x2& a, const f2x2& b)
{
    return {make_float2(__fadd_rn(a.lo.x, b.lo.x), __fadd_rn(a.lo.y, b.lo.y)), make_float2(__fadd_rn(a.hi.x, b.hi.x), __fadd_rn(a.hi.y, b.hi.y))};
}
__device__ __forceinline__ float get(const f2x2& v, int j) { return j == 0 ? v.lo.x : (j == 1 ? v.lo.y : (j == 2 ? v.hi.x : v.hi.y)); }

// PSM_KNOCKOUT (never defined in the product build): an experiment may compile this header with single operation
// classes removed -- results are wrong, only the TIME is of interest -- to measure what the kernel is sensitive to.
// bit 0 shuffles, bit 1 history ring, bit 2 guide loads, bit 3 stores, bit 4 stage-1 widening + fp64 running sums,
// bit 5 volume (p) loads.
#ifndef PSM_KNOCKOUT
#define PSM_KNOCKOUT 0
#endif
__device__ __forceinline__ float4 ko_fake(const char* p)
{
    const float f = __int_as_float(0x3f000000 | ((int)(size_t)p & 0xffff));
    return make_float4(f, f, f, f);
}
__device__ __forceinline__ float4 ldg4(const char* __restrict__ p)    // volume rows
{
    if (PSM_KNOCKOUT & 32) return ko_fake(p);
    return __ldg(reinterpret_cast<const float4*>(p));
}
__device__ __forceinline__ float4 ldg4g(const char* __restrict__ p)   // guide rows
{
    if (PSM_KNOCKOUT & 4) return ko_fake(p);
    return __ldg(reinterpret_cast<const float4*>(p));
}

__device__ __forceinline__ void prefetch_l1(const char* p) { asm volatile("prefetch.global.L1 [%0];" :: "l"(p)); }

__device__ __forceinline__ unsigned umax4(const float4& v)
{
    return max(max(__float_as_uint(v.x), __float_as_uint(v.y)), max(__float_as_uint(v.z), __float_as_uint(v.w)));
}

// fp32 8-wide window sums from the 4 column sums a lane owns (MIXED stage 2), same tree as hsum8
__device__ __forceinline__ f2x2 hsum8f(const f2x2& c)
{
    const float c0 = c.lo.x, c1 = c.lo.y, c2 = c.hi.x, c3 = c.hi.y;
    const float P2 = __fadd_rn(c0, c1), P3 = __fadd_rn(P2, c2), Tt = __fadd_rn(P3, c3);
    const float S2 = __fadd_rn(c2, c3), S3 = __fadd_rn(c1, S2);
#if PSM_KNOCKOUT & 1
    const float Tn = Tt, Q1 = c0, Q2 = P2, Q3 = P3;
#else
    const float Tn = __shfl_down_sync(0xffffffffu, Tt, 1);
    const float Q1 = __shfl_down_sync(0xffffffffu, c0, 2);
    const float Q2 = __shfl_down_sync(0xffffffffu, P2, 2);
    const float Q3 = __shfl_down_sync(0xffffffffu, P3, 2);
#endif
    f2x2 h;
    h.lo.x = __fadd_rn(Tt, Tn);
    h.lo.y = __fadd_rn(__fadd_rn(S3, Tn), Q1);
    h.hi.x = __fadd_rn(__fadd_rn(S2, Tn), Q2);
    h.hi.y = __fadd_rn(__fadd_rn(c3, Tn), Q3);
    return h;
}


// ---- TMA (bulk async copy) staging of the guide rows --------------------------------------------
// The 13 guide rows a step needs (10 coefficient planes at the a,b columns, 3 image planes at the
// input columns) are identical for every slice-warp of a CTA.  One elected lane of warp 0 copies them
// global -> shared with cp.async.bulk (the TMA engine; one 512/544-byte row per instruction) two steps
// ahead; completion is signalled on an mbarrier (complete_tx), consumption on a second mbarrier with
// one arrival per warp.  Consumers read with LDS at immediate offsets: no per-load address arithmetic,
// no L2 latency on the critical path, and the image rows (needed as newest, output and oldest row of
// the stage-1 window) stay in a 16-row ring, so they are fetched from L2 once per CTA instead of
// three times per warp.  The staging area lies in front of the rings in the dynamic shared memory.
constexpr int kStCoefStages = 4;       // coefficient stages in flight (power of two)
constexpr int kStIRows = 16;           // image-row ring (power of two >= 8 + stages)
constexpr int kStLook = 2;             // the producer runs this many steps ahead
constexpr int kStIRowFloats = 136;     // 128 input columns + 8 so that the output columns (+8) stay inside the row
constexpr int kStBarBytes = 128;
constexpr int kStCoefBytes = kStCoefStages * 10 * 128 * 4;
constexpr int kStIBytes = kStIRows * 3 * kStIRowFloats * 4;
constexpr int kStSmemBytes = kStBarBytes + kStCoefBytes + kStIBytes;

__device__ __forceinline__ void mbar_init(unsigned bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes) { asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory"); }
__device__ __forceinline__ void mbar_arrive(unsigned bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
{
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra WAIT_DONE;\n\tbra WAIT_LOOP;\n\tWAIT_DONE:\n\t}"
                 :: "r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(unsigned dst, const void* src, unsigned bytes, unsigned bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ float4 lds4(unsigned addr)
{
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}

// MINB: resident CTAs per SM the register allocation is sized for (3 -> <=168 regs, 4 -> <=128);
// IW  : 0 = F2F everywhere; 1 = integer widening into the scaled domain in both stages; 2 = integer widening in
//       stage 1 (non-negative values: one instruction each), F2F in the exact stage 2 (signed values would cost three)
// S2M : kS2Exact / kS2Mixed
// PA  : 1 = adds / subtracts of products as fma with a run-time unit multiplier (exact, see fma2)
// PF  : 1 = prefetch the next step's guide rows into L1;  2 = stage the guide rows in shared memory with bulk async
//       copies (TMA) issued two steps ahead by one lane per CTA;
//       3 = light prefetch (only the newest p row a step ahead; everything else is loaded where it is used);
//       4 = the ten coefficient rows are loaded one step ahead as well (40 more live registers)
// register budgets by MINB: 3 -> 168 regs (3 CTAs x 128 thr or 4 x 96: 12 warps/SM); 4 -> 128 regs; 5 -> 144 regs
// (2 CTAs x 224 thr = 14 warps); 6 -> 152 regs.  Shared memory (512 B of ring per thread) caps an SM at 3 CTAs of 128.
constexpr int cvf_max_regs(int minb) { return minb == 3 ? 168 : (minb == 4 ? 128 : (minb == 5 ? 144 : 152)); }

template <int MINB, int IW, int S2M, int PF = 0, int PA = 0>
__global__ void __maxnreg__(cvf_max_regs(MINB))
cvf_stream_kernel(const CvfParams P)
{
    extern __shared__ float4 smem_dyn[];  // PF == 2: staging area (kStSmemBytes), then the rings
    float4* ring = smem_dyn + (PF == 2 ? kStSmemBytes / 16 : 0);  // [8 slots][4 planes][blockDim.x threads]
    constexpr bool MIXED = (S2M == kS2Mixed);
    constexpr double kMean1 = IW ? kMeanScaled : kMeanPlain;   // stage-1 mean scale
    constexpr double kMean2 = IW == 1 ? kMeanScaled : kMeanPlain;   // stage-2 (exact) mean scale: IW == 2 keeps S2 unscaled
    const int tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int nthr = blockDim.x;
    const int wpc = nthr >> 5;
    const float2 kOne2 = make_float2(P.one, P.one), kMone2 = make_float2(P.mone, P.mone);
    auto xadd = [&](const f2x2& a, const f2x2& b) -> f2x2 {   // a + b, exact, b or a may be products
        if (PA) return {fma2(a.lo, kOne2, b.lo), fma2(a.hi, kOne2, b.hi)};
        return add2(a, b);
    };
    auto xsub = [&](const f2x2& a, const f2x2& b) -> f2x2 {   // a - b
        if (PA) return {fma2(b.lo, kMone2, a.lo), fma2(b.hi, kMone2, a.hi)};
        return sub2(a, b);
    };

    // Block -> work mapping.  Hardware hands consecutive blockIdx to consecutive SMs, so the CTAs that
    // share an SM (and its L1) are blockIdx k, k+nsm, k+2nsm, ...; the remap makes those neighbours in
    // work order (consecutive slice groups of the same strip and segment), which read the same guide rows.
    int b = blockIdx.x;
    const bool packed = P.pack_gl > 0 && b >= P.pack_first;
    if (P.remap_sms > 0) {
        const int per = P.remap_sms * P.remap_ctas;
        const int chunk = b / per, r = b - chunk * per;
        if ((chunk + 1) * per <= (int)gridDim.x) b = chunk * per + (r % P.remap_sms) * P.remap_ctas + r / P.remap_sms;
    }
    int dgroup, strip, seg, view;
    if (packed) {
        b -= P.pack_first;
        dgroup = b % P.pack_ndg; b /= P.pack_ndg;
        strip = P.nstrips;     // the remainder: one past the regular strips
        seg = b % P.nseg;
        view = b / P.nseg;
    } else {
        dgroup = b % P.ndgroups; b /= P.ndgroups;
        strip = b % P.nstrips;   b /= P.nstrips;
        seg = b % P.nseg;
        view = b / P.nseg;
    }
    const int gl = packed ? P.pack_gl : 32;   // lanes per slice
    const int gln = lane & (gl - 1);          // lane within its slice group
    const int gbase = lane - gln;
    const int dlc_raw = packed ? (dgroup * wpc + warp) * (32 / gl) + lane / gl : dgroup * wpc + warp;
    const bool active = dlc_raw < P.Dloc;     // warp-uniform unless packed
    const int dlc = active ? dlc_raw : P.Dloc - 1;
    constexpr bool ST = (PF == 2);
    const unsigned st_base = (unsigned)__cvta_generic_to_shared(smem_dyn);   // staging area (ST): barriers, coefficient stages, image-row ring
    if (ST) {
        if (tid == 0) {
#pragma unroll
            for (int i = 0; i < kStCoefStages; ++i) { mbar_init(st_base + 8 * i, 1); mbar_init(st_base + 8 * (kStCoefStages + i), wpc); }
            mbar_init(st_base + 8 * 2 * kStCoefStages, 1);   // prologue barrier
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
        __syncthreads();   // the barriers are initialised before anyone waits on them; the only CTA-wide synchronisation
        // a surplus warp of the last slice group (Dloc % wpc != 0) redoes the last slice with its stores masked:
        // every warp arrives on the stage barriers
    } else if (!__any_sync(0xffffffffu, active)) {
        return;  // warps never synchronise with each other; lanes of a packed warp do (shuffles), so only whole warps leave
    }

    const int W = P.W, H = P.H;
    const unsigned Wp = (unsigned)P.Wp;
    const unsigned plane = (unsigned)H * Wp;
    const int out_lo = strip * kStripOut;
    const int X0 = packed ? P.pack_x0
                          : ((P.pack_gl == 0 && strip == P.nstrips - 1 && strip > 0) ? ((W - kStripOut + 3) & ~3) : out_lo);
    const int cin = X0 - 8 + 4 * gln;
    // per-thread base pointers (bytes); every offset added to them below is warp-uniform
    const char* __restrict__ Gi = reinterpret_cast<const char*>(P.guide[view] + cin);      // guide, input columns
    const char* __restrict__ Ga = reinterpret_cast<const char*>(P.guide[view] + cin + 4);  // guide, a,b columns
    const char* __restrict__ Go = reinterpret_cast<const char*>(P.guide[view] + cin + 8);  // guide, output columns
    const char* __restrict__ vin = reinterpret_cast<const char*>(P.vol_in[view] + (size_t)dlc * plane + cin);
    char* __restrict__ vout = reinterpret_cast<char*>(P.vol_out[view] + (size_t)dlc * plane + cin + 8);
    const size_t planeB = (size_t)plane * 4, rowB = (size_t)Wp * 4;
    const bool store_ok = active && gln <= gl - 5 && cin + 8 < W && cin + 8 >= out_lo;

    // a guide with negative / non-finite values (outside the [0,1] image contract) disables the
    // integer widening for the whole launch of this view; `slow` also turns sticky once a row of p
    // needed the slow path, so that non-finite a,b are widened by F2F as well
    bool slow = IW ? (__ldg(P.guide_flags + view) != 0) : true;

    // ---- x-reflection plan for a,b (strips whose a,b columns X0-4 .. X0+115 leave the image) ----
    const bool fix_left = X0 == 0;
    const bool fix_right = X0 + 4 * gl - 13 >= W;   // last valid a,b column of the (group's) strip
    int fix_src[4];               // source lane of element j (this lane's a,b column X0-4+4l+j mirrored into the image)
    unsigned maskL = 0, maskR = 0;  // bit j: element j lies left of column 0 / right of column W-1
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int xa = cin + 4 + j;
        const int r = reflect101(xa < -4 ? -4 : (xa > W + 2 ? W + 2 : xa), W) - (X0 - 4);
        fix_src[j] = gbase + ((r >> 2) & (gl - 1));
        maskL |= (fix_left && xa < 0) ? (1u << j) : 0u;
        maskR |= (fix_right && xa >= W && xa <= W + 2) ? (1u << j) : 0u;
    }
    // which element of the source lane: left (8-j)&3, right (2(W-1)-j)&3 -- uniform per side, so the
    // source lane (which does not know who reads it) can put the right element on the wire
    const int eR = (2 * (W - 1)) & 3;

    const int Y0 = seg * P.seg_rows;
    const int Y1 = min(H, Y0 + P.seg_rows);
    const bool top = (Y0 == 0);
    const bool bottom = (Y1 == H);
    const int T0 = top ? 0 : Y0 - 4;              // first a,b row
    const int Tlast = bottom ? H - 1 : Y1 + 2;    // last real a,b row
    const int Tend = bottom ? H + 2 : Tlast;      // last step (three virtual rows below the image)

    double S1[4][4];
    double S2[MIXED ? 1 : 4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int j = 0; j < 4; ++j) { S1[q][j] = 0.0; S2[MIXED ? 0 : q][j] = 0.0; }

    // history ring accessors (slot = 0..7): a whole slot = 4 planes x 4 columns of this thread
    auto ring_ld = [&](int slot, f2x2 (&v)[4]) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            if (PSM_KNOCKOUT & 2) v[q] = {make_float2(1.f, 2.f), make_float2(3.f, (float)slot)};
            else v[q] = from4(ring[(slot * 4 + q) * nthr + tid]);
        }
    };
    auto ring_st = [&](int slot, const f2x2 (&v)[4]) {
        if (PSM_KNOCKOUT & 2) return;
#pragma unroll
        for (int q = 0; q < 4; ++q) ring[(slot * 4 + q) * nthr + tid] = to4(v[q]);
    };
    auto ring_wait_ld = [&]() {};
    auto ring_wait_st = [&]() {};

    struct RowIn { float4 p, i0, i1, i2; };
    auto load_at = [&](size_t ro) {  // ro: byte offset of the row
        RowIn x;
        x.p = ldg4(vin + ro);
        x.i0 = ldg4g(Gi + ro);
        x.i1 = ldg4g(Gi + (planeB + ro));
        x.i2 = ldg4g(Gi + (2 * planeB + ro));
        return x;
    };
    auto load_row = [&](int r) { return load_at((size_t)reflect101(r, H) * rowB); };
    // warp-uniform: true when some lane's p holds a negative (incl. -0), inf, nan or >= 2^63 value (the guide is
    // < 2^63 when its flag is clear, so every product I * p that the fast path widens is finite)
    auto needs_slow = [&](const float4& pa, const float4& pb) {
        return __any_sync(0xffffffffu, max(umax4(pa), umax4(pb)) >= 0x5f000000u) != 0;
    };
    // S1 += / -= one input row.  WID: 0 F2F unscaled, 1 integer non-negative (scaled), 2 F2F scaled
    auto acc_row = [&](const RowIn& x, auto wid_tag, auto sub_tag) {
        constexpr int WID = decltype(wid_tag)::value;
        constexpr bool SUB = decltype(sub_tag)::value;
        if (PSM_KNOCKOUT & 16) { S1[0][0] = __hiloint2double(__float_as_int(x.p.x), __float_as_int(x.i0.y)); return; }
        const f2x2 p = from4(x.p);
        const f2x2 m0 = mul2(from4(x.i0), p), m1 = mul2(from4(x.i1), p), m2 = mul2(from4(x.i2), p);  // CVF.cpp:87
        auto w = [](float f) { return WID == 0 ? (double)f : (WID == 1 ? widen_nn(f) : widen_any(f)); };
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            if (SUB) {
                S1[0][j] = __dsub_rn(S1[0][j], w(get(p, j)));
                S1[1][j] = __dsub_rn(S1[1][j], w(get(m0, j)));
                S1[2][j] = __dsub_rn(S1[2][j], w(get(m1, j)));
                S1[3][j] = __dsub_rn(S1[3][j], w(get(m2, j)));
            } else {
                S1[0][j] = __dadd_rn(S1[0][j], w(get(p, j)));
                S1[1][j] = __dadd_rn(S1[1][j], w(get(m0, j)));
                S1[2][j] = __dadd_rn(S1[2][j], w(get(m1, j)));
                S1[3][j] = __dadd_rn(S1[3][j], w(get(m2, j)));
            }
        }
    };
    using I0 = std::integral_constant<int, 0>;
    using I1 = std::integral_constant<int, 1>;
    using I2 = std::integral_constant<int, 2>;
    using Tadd = std::false_type;
    using Tsub = std::true_type;
    auto add_row = [&](const RowIn& x, bool slow_row) {
        if (!IW) acc_row(x, I0{}, Tadd{});
        else if (slow_row) acc_row(x, I2{}, Tadd{});
        else acc_row(x, I1{}, Tadd{});
    };
    auto sub_row = [&](const RowIn& x, bool slow_row) {
        if (!IW) acc_row(x, I0{}, Tsub{});
        else if (slow_row) acc_row(x, I2{}, Tsub{});
        else acc_row(x, I1{}, Tsub{});
    };
    auto load_guide = [&](size_t ro, float4 (&g4)[10]) {
#pragma unroll
        for (int q = 0; q < 10; ++q) g4[q] = ldg4g(Ga + ((size_t)(kGuideMean + q) * planeB + ro));
    };
    auto mean4 = [](const double (&h)[4], double scale) {
        f2x2 m;
        m.lo = make_float2((float)__dmul_rn(h[0], scale), (float)__dmul_rn(h[1], scale));
        m.hi = make_float2((float)__dmul_rn(h[2], scale), (float)__dmul_rn(h[3], scale));
        return m;
    };

    // stage-1 row sums -> means -> cov -> a,b (CVF.cpp:81-155), then the x-reflection of a,b
    auto coeffs = [&](const float4 (&g4)[10], f2x2 (&av)[4]) {
        f2x2 m[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            double h[4];
            hsum8(S1[q], h);
            m[q] = mean4(h, kMean1);
        }
        const f2x2 mI0 = from4(g4[0]), mI1 = from4(g4[1]), mI2 = from4(g4[2]);
        const f2x2 M00 = from4(g4[3]), M01 = from4(g4[4]), M02 = from4(g4[5]);
        const f2x2 M11 = from4(g4[6]), M12 = from4(g4[7]), M22 = from4(g4[8]);
        const f2x2 idet = from4(g4[9]);
        const f2x2 c0 = xsub(m[1], mul2(mI0, m[0]));   // CVF.cpp:92-95
        const f2x2 c1 = xsub(m[2], mul2(mI1, m[0]));
        const f2x2 c2 = xsub(m[3], mul2(mI2, m[0]));
        av[0] = mul2(idet, xadd(xadd(mul2(c0, M00), mul2(c1, M01)), mul2(c2, M02)));  // CVF.cpp:121-146
        av[1] = mul2(idet, xadd(xadd(mul2(c0, M01), mul2(c1, M11)), mul2(c2, M12)));
        av[2] = mul2(idet, xadd(xadd(mul2(c0, M02), mul2(c1, M12)), mul2(c2, M22)));
        av[3] = xsub(xsub(xsub(m[0], mul2(av[0], mI0)), mul2(av[1], mI1)), mul2(av[2], mI2));  // CVF.cpp:152-155
        if (fix_left | fix_right) {  // warp-uniform
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float e[4] = {av[q].lo.x, av[q].lo.y, av[q].hi.x, av[q].hi.y};
                float r[4] = {e[0], e[1], e[2], e[3]};
                if (fix_left) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float v = __shfl_sync(0xffffffffu, e[(8 - j) & 3], fix_src[j]);
                        if ((maskL >> j) & 1u) r[j] = v;
                    }
                }
                if (fix_right) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const int er = (eR - j) & 3;
                        const float sv = er == 0 ? e[0] : (er == 1 ? e[1] : (er == 2 ? e[2] : e[3]));
                        const float v = __shfl_sync(0xffffffffu, sv, fix_src[j]);
                        if ((maskR >> j) & 1u) r[j] = v;
                    }
                }
                av[q] = {make_float2(r[0], r[1]), make_float2(r[2], r[3])};
            }
        }
    };

    // q = box(b) + box(a0)*I0 + box(a1)*I1 + box(a2)*I2, accumulated in that order (CVF.cpp:157-163)
    auto combine = [&](size_t ro, const f2x2 (&mb)[4], const float4& i0, const float4& i1, const float4& i2) {
        f2x2 qv = xadd(mb[3], mul2(mb[0], from4(i0)));
        qv = xadd(qv, mul2(mb[1], from4(i1)));
        qv = xadd(qv, mul2(mb[2], from4(i2)));
        if (store_ok && !((PSM_KNOCKOUT & 8) && qv.lo.x != 12345.f)) *reinterpret_cast<float4*>(vout + ro) = to4(qv);
    };
    // EXACT: stage-2 row sums of S2 -> q for one output row
    auto emit = [&](size_t ro, const float4& i0, const float4& i1, const float4& i2) {
        f2x2 mb[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            double h2[4];
            hsum8(S2[MIXED ? 0 : q], h2);
            mb[q] = mean4(h2, kMean2);
        }
        combine(ro, mb, i0, i1, i2);
    };
    // MIXED: the two half-window sums  P(y-3)+P(y-1)  and  P(y+1)+P(y+3)  -> q for one output row
    auto emit_pairs = [&](size_t ro, const f2x2 (&lo)[4], const f2x2 (&hi)[4],
                          const float4& i0, const float4& i1, const float4& i2) {
        f2x2 mb[4];
        const f2x2 k64 = {make_float2(1.f / 64.f, 1.f / 64.f), make_float2(1.f / 64.f, 1.f / 64.f)};
#pragma unroll
        for (int q = 0; q < 4; ++q) mb[q] = mul2(hsum8f(addp(lo[q], hi[q])), k64);
        combine(ro, mb, i0, i1, i2);
    };
    // widening of a,b values for the exact stage 2
    auto w2 = [&](float f, bool slow_now) { return IW != 1 ? (double)f : (slow_now ? widen_any(f) : widen_sg(f)); };

    // MIXED: pair-row index with the row reflection folded in: P(s) = pair(refl_p(s))
    auto refl_p = [&](int s) { return s <= 0 ? 1 - s : (s >= H ? 2 * H - 1 - s : s); };

    // ---- generic step: any row, every special case (top weights, warm-up, reflection, virtual rows)
    auto generic_step = [&](int t) {
        const bool real_row = t <= Tlast;
        f2x2 av[4];
        if (real_row) {
            const RowIn xn = load_row(t + 3);
            const RowIn xo = load_row(t - 4);
            float4 g4[10];
            load_guide((size_t)t * rowB, g4);
            const bool slow_row = slow || (IW && needs_slow(xn.p, xo.p));
            slow = slow_row;   // sticky
            add_row(xn, slow_row);
            coeffs(g4, av);
            sub_row(xo, slow_row);
        }
        const int age = t - T0;
        const bool warm = top ? (t <= 4) : (age < 8);
        const bool first_out = top ? (t == 4) : (age == 7);
        if (!MIXED) {
            ring_wait_st();
            if (!real_row) {  // virtual a,b row below the image == reflected row, still in the ring
                ring_ld(reflect101(t, H) & 7, av);
                ring_wait_ld();
            }
            const double wnew = (top && t >= 1 && t <= 3) ? 2.0 : 1.0;      // rows 1..3 appear twice in row 0's window
            const int oslot = (top && t < 8) ? ((8 - t) & 7) : (t & 7);      // slot of a,b row reflect(t-8)
            const int nslot = t & 7;
            f2x2 old[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) old[q] = {make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
            if (!warm) { ring_ld(oslot, old); ring_wait_ld(); }
            if (real_row) ring_st(nslot, av);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    double s = __fma_rn(wnew, w2(get(av[q], j), slow), S2[MIXED ? 0 : q][j]);  // exact: wnew is 1 or 2
                    if (!warm) s = __dsub_rn(s, w2(get(old[q], j), slow));
                    S2[MIXED ? 0 : q][j] = s;
                }
            }
        } else if (real_row) {
            // MIXED ring protocol: slot t&7 holds ab(t-1) until pair(t) = ab(t-1) + ab(t) replaces it; ab(t) waits in
            // slot (t+1)&7, which is dead (pair(t-7) was last read at step t-1).  No a,b row lives in registers.
            ring_wait_st();
            if (t > T0) {  // the first row of a segment has no predecessor
                f2x2 pr[4];
                ring_ld(t & 7, pr);
                ring_wait_ld();
#pragma unroll
                for (int q = 0; q < 4; ++q) pr[q] = xadd(av[q], pr[q]);
                ring_st(t & 7, pr);
            }
            ring_st((t + 1) & 7, av);
        }
        if (warm && !first_out) return;
        const int nrows = (top && t == 4) ? 2 : 1;  // output rows 0 and 1 share one reflected window
        for (int e = 0; e < nrows; ++e) {
            const int y = (top && t == 4) ? e : t - 3;
            if (y < Y0 || y >= Y1) continue;
            const size_t ro = (size_t)y * rowB;
            const float4 o0 = ldg4g(Go + ro), o1 = ldg4g(Go + (planeB + ro)), o2 = ldg4g(Go + (2 * planeB + ro));
            if (!MIXED) {
                emit(ro, o0, o1, o2);
            } else {
                f2x2 pa[4], pb[4], pc[4], pd[4];
                ring_wait_st();
                ring_ld(refl_p(y - 3) & 7, pa);
                ring_ld(refl_p(y - 1) & 7, pb);
                ring_ld(refl_p(y + 1) & 7, pc);
                ring_ld(refl_p(y + 3) & 7, pd);
                ring_wait_ld();
#pragma unroll
                for (int q = 0; q < 4; ++q) { pa[q] = addp(pa[q], pb[q]); pc[q] = addp(pc[q], pd[q]); }
                emit_pairs(ro, pa, pc, o0, o1, o2);
            }
        }
    };

    // ---- schedule ----------------------------------------------------------------------------
    // steady steps need: a real row, no warm-up, no reflected input row (t-4 >= 0, t+4 <= H-1 because
    // the step also preloads row t+4 for its successor) and the plain ring slot t&7
    const int Ts0 = top ? 8 : T0 + 8;
    const int Ts1 = min(Tlast, H - 5);

    for (int r = T0 - 4; r <= T0 + 2; ++r) {
        const RowIn x = load_row(r);
        const bool slow_row = slow || (IW && needs_slow(x.p, x.p));
        slow = slow_row;
        add_row(x, slow_row);
    }
    int t = T0;
    for (; t <= Tend && t < Ts0; ++t) generic_step(t);

    if (t <= Ts1) {
        size_t ro_n = (size_t)(t + 3) * rowB;  // newest input row  t+3   (byte offsets)
        size_t ro_o = (size_t)(t - 4) * rowB;  // oldest input row  t-4
        size_t ro_t = (size_t)t * rowB;        // a,b row           t
        size_t ro_y = (size_t)(t - 3) * rowB;  // output row        t-3
        RowIn xn = load_at(ro_n);   // newest row of the next stage-1 step (loaded one step ahead)
        RowIn xo = load_at(ro_o);   // oldest row of the next stage-1 step (loaded one step ahead)
        // One steady step.  SLOW (compile time) selects the F2F widening for rows outside the integer
        // domain; the fast loop below leaves for the slow loop the first time a vote says so and never
        // comes back (sticky), so the fast loop is straight-line code.
        float4 g4n[PF == 4 ? 10 : 1];   // PF == 4: the coefficient rows of the NEXT step, loaded right after this step's were consumed
        if (PF == 4) {
#pragma unroll
            for (int q = 0; q < (PF == 4 ? 10 : 1); ++q) g4n[q] = ldg4(Ga + ((size_t)(kGuideMean + q) * planeB + ro_t));
        }
        auto steady = [&](auto slow_tag) {
            constexpr bool SLOW = decltype(slow_tag)::value;
            const float4 o0 = ldg4g(Go + ro_y), o1 = ldg4g(Go + (planeB + ro_y)), o2 = ldg4g(Go + (2 * planeB + ro_y));
            f2x2 av[4];
            {   // stage 1 of a,b row ro_t: S1 += newest, row sums -> a,b, S1 -= oldest; refills xn / xo
                float4 g4[10];
                if (PF == 4) {
#pragma unroll
                    for (int q = 0; q < 10; ++q) g4[q] = g4n[PF == 4 ? q : 0];
                } else load_guide(ro_t, g4);
                if (PF) {   // next step's coefficient rows and output-column guide rows -> L1 (one step = thousands of cycles ahead)
#pragma unroll
                    for (int q = 0; q < 10; ++q) prefetch_l1(Ga + ((size_t)(kGuideMean + q) * planeB + ro_t + rowB));
#pragma unroll
                    for (int q = 0; q < 3; ++q) prefetch_l1(Go + ((size_t)q * planeB + ro_y + rowB));
                }
                add_row(xn, SLOW);
                ro_n += rowB;
                xn = load_at(ro_n);     // into the registers add_row just released
                coeffs(g4, av);
                if (PF == 4) {   // next step's coefficient rows: a whole stage 2 (and the tail of stage 1) ahead of their first use
#pragma unroll
                    for (int q = 0; q < (PF == 4 ? 10 : 1); ++q) g4n[q] = ldg4(Ga + ((size_t)(kGuideMean + q) * planeB + ro_t + rowB));
                }
                sub_row(xo, SLOW);
                ro_o += rowB;
                xo = load_at(ro_o);
                ro_t += rowB;
            }
            if (!MIXED) {
                // stage 2 (exact) of a,b row t (output row t-3): ring exchange, S2 update, q
                f2x2 old[4];
                ring_wait_st();
                ring_ld(t & 7, old);
                ring_wait_ld();
                ring_st(t & 7, av);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
#pragma unroll
                    for (int j = 0; j < 4; ++j)
                        S2[MIXED ? 0 : q][j] = __dsub_rn(__dadd_rn(S2[MIXED ? 0 : q][j], w2(get(av[q], j), SLOW)), w2(get(old[q], j), SLOW));
                }
                emit(ro_y, o0, o1, o2);
            } else {
                // stage 2 (mixed): pair(t) into the ring, window = (pair(t-6)+pair(t-4)) + (pair(t-2)+pair(t))
                f2x2 pa[4], pb[4], pc[4], pd[4];
                ring_wait_st();
                ring_ld((t - 6) & 7, pa);
                ring_ld((t - 4) & 7, pb);
                ring_wait_ld();
#pragma unroll
                for (int q = 0; q < 4; ++q) pa[q] = addp(pa[q], pb[q]);          // P(y-3) + P(y-1)
                ring_ld((t - 2) & 7, pc);
                ring_ld(t & 7, pd);                                              // ab(t-1)
                ring_wait_ld();
#pragma unroll
                for (int q = 0; q < 4; ++q) pd[q] = xadd(av[q], pd[q]);          // pair(t): scalar adds (av are products)
                ring_st(t & 7, pd);
                ring_st((t + 1) & 7, av);
#pragma unroll
                for (int q = 0; q < 4; ++q) pc[q] = addp(pc[q], pd[q]);          // P(y+1) + P(y+3)
                emit_pairs(ro_y, pa, pc, o0, o1, o2);
            }
            ro_y += rowB;
        };
        if (PF == 3) {
            // ---- "light prefetch" steady loop: only the NEWEST p row (which comes from HBM) is loaded a step ahead; the
            // image rows, the oldest p row (read 7 steps ago by this warp) and the coefficient rows are mostly cache hits
            // and are loaded where they are used.
            // 28 fewer live registers than the full prefetch: the build for 16 warps per SM (<= 128 registers).
            float4 pn = xn.p;
            auto steady_lp = [&](auto slow_tag) {
                constexpr bool SLOW = decltype(slow_tag)::value;
                f2x2 av[4];
                {
                    float4 g4[10];
                    load_guide(ro_t, g4);
                    RowIn x;
                    x.p = pn; x.i0 = ldg4(Gi + ro_n); x.i1 = ldg4(Gi + (planeB + ro_n)); x.i2 = ldg4(Gi + (2 * planeB + ro_n));
                    add_row(x, SLOW);
                    ro_n += rowB;
                    pn = ldg4(vin + ro_n);
                    coeffs(g4, av);
                    const RowIn xold = load_at(ro_o);
                    sub_row(xold, SLOW);
                    ro_o += rowB;
                    ro_t += rowB;
                }
                const float4 o0 = ldg4g(Go + ro_y), o1 = ldg4g(Go + (planeB + ro_y)), o2 = ldg4g(Go + (2 * planeB + ro_y));
                if (!MIXED) {
                    f2x2 old[4];
                    ring_wait_st();
                    ring_ld(t & 7, old);
                    ring_wait_ld();
                    ring_st(t & 7, av);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            S2[MIXED ? 0 : q][j] = __dsub_rn(__dadd_rn(S2[MIXED ? 0 : q][j], w2(get(av[q], j), SLOW)), w2(get(old[q], j), SLOW));
                    }
                    emit(ro_y, o0, o1, o2);
                } else {
                    f2x2 pa[4], pb[4], pc[4], pd[4];
                    ring_wait_st();
                    ring_ld((t - 6) & 7, pa);
                    ring_ld((t - 4) & 7, pb);
                    ring_wait_ld();
#pragma unroll
                    for (int q = 0; q < 4; ++q) pa[q] = addp(pa[q], pb[q]);
                    ring_ld((t - 2) & 7, pc);
                    ring_ld(t & 7, pd);
                    ring_wait_ld();
#pragma unroll
                    for (int q = 0; q < 4; ++q) pd[q] = xadd(av[q], pd[q]);
                    ring_st(t & 7, pd);
                    ring_st((t + 1) & 7, av);
#pragma unroll
                    for (int q = 0; q < 4; ++q) pc[q] = addp(pc[q], pd[q]);
                    emit_pairs(ro_y, pa, pc, o0, o1, o2);
                }
                ro_y += rowB;
            };
            if (IW) {
                for (; t <= Ts1 && !slow; ++t) {
                    if (needs_slow(pn, pn)) { slow = true; break; }   // the oldest row was checked when it was the newest
                    steady_lp(std::false_type{});
                }
            }
            for (; t <= Ts1; ++t) steady_lp(std::true_type{});
        } else if (!ST) {
            if (IW) {
                for (; t <= Ts1 && !slow; ++t) {
                    if (needs_slow(xn.p, xo.p)) { slow = true; break; }
                    steady(std::false_type{});
                }
            }
            for (; t <= Ts1; ++t) steady(std::true_type{});
        } else {
            // ---- steady loop with TMA-staged guide rows -------------------------------------------------
            const int t_s = t, klast = Ts1 - t_s;
            const unsigned bar_full = st_base, bar_empty = st_base + 8 * kStCoefStages, bar_pro = st_base + 8 * 2 * kStCoefStages;
            const unsigned coef_s = st_base + kStBarBytes, iring_s = coef_s + kStCoefBytes;
            const float* gbase = P.guide[view];
            const unsigned lane16 = (unsigned)lane * 16u;
            auto issue = [&](int k) {   // one lane: the 13 rows of step k -> stage k & 3 / image-row slot (t_s+k+3) & 15
                const int sidx = k & (kStCoefStages - 1);
                const unsigned bar = bar_full + 8 * sidx;
                const int tt = t_s + k;
                mbar_expect_tx(bar, 10 * 512 + 3 * kStIRowFloats * 4);
#pragma unroll
                for (int q = 0; q < 10; ++q)
                    bulk_g2s(coef_s + (unsigned)((sidx * 10 + q) * 512), gbase + (size_t)(kGuideMean + q) * plane + (size_t)tt * Wp + (X0 - 4), 512, bar);
                const int ri = tt + 3;
#pragma unroll
                for (int c3 = 0; c3 < 3; ++c3)
                    bulk_g2s(iring_s + (unsigned)((((ri & (kStIRows - 1)) * 3 + c3) * kStIRowFloats) * 4),
                             gbase + (size_t)c3 * plane + (size_t)ri * Wp + (X0 - 8), kStIRowFloats * 4, bar);
            };
            if (warp == 0 && lane == 0) {   // prologue: image rows t_s-4 .. t_s+2 and the first kStLook stages
                mbar_expect_tx(bar_pro, 7 * 3 * kStIRowFloats * 4);
                for (int ri = t_s - 4; ri <= t_s + 2; ++ri)
#pragma unroll
                    for (int c3 = 0; c3 < 3; ++c3)
                        bulk_g2s(iring_s + (unsigned)((((ri & (kStIRows - 1)) * 3 + c3) * kStIRowFloats) * 4),
                                 gbase + (size_t)c3 * plane + (size_t)ri * Wp + (X0 - 8), kStIRowFloats * 4, bar_pro);
                for (int k = 0; k < kStLook && k <= klast; ++k) issue(k);
            }
            mbar_wait(bar_pro, 0);
            auto irow = [&](int r) { return iring_s + (unsigned)(((r & (kStIRows - 1)) * 3 * kStIRowFloats) * 4) + lane16; };
            auto steady_st = [&](auto slow_tag) {
                constexpr bool SLOW = decltype(slow_tag)::value;
                const int k = t - t_s;
                if (warp == 0 && k + kStLook <= klast) {   // producer: refill the stage that every warp released four steps ago
                    const int kk = k + kStLook;
                    if (kk >= kStCoefStages) mbar_wait(bar_empty + 8 * (kk & (kStCoefStages - 1)), ((kk >> 2) + 1) & 1);
                    if (lane == 0) issue(kk);
                    __syncwarp();
                }
                mbar_wait(bar_full + 8 * (k & (kStCoefStages - 1)), (k >> 2) & 1);
                f2x2 av[4];
                {
                    const unsigned cs = coef_s + (unsigned)((k & (kStCoefStages - 1)) * 10 * 512) + lane16;
                    const unsigned inew = irow(t + 3), iold = irow(t - 4);
                    RowIn x;
                    x.p = xn.p; x.i0 = lds4(inew); x.i1 = lds4(inew + kStIRowFloats * 4); x.i2 = lds4(inew + 2 * kStIRowFloats * 4);
                    add_row(x, SLOW);
                    ro_n += rowB;
                    xn.p = ldg4(vin + ro_n);
                    float4 g4[10];
#pragma unroll
                    for (int q = 0; q < 10; ++q) g4[q] = lds4(cs + q * 512);
                    coeffs(g4, av);
                    x.p = xo.p; x.i0 = lds4(iold); x.i1 = lds4(iold + kStIRowFloats * 4); x.i2 = lds4(iold + 2 * kStIRowFloats * 4);
                    sub_row(x, SLOW);
                    ro_o += rowB;
                    xo.p = ldg4(vin + ro_o);
                }
                const unsigned iout = irow(t - 3) + 32u;   // output columns = input columns + 8
                const float4 o0 = lds4(iout), o1 = lds4(iout + kStIRowFloats * 4), o2 = lds4(iout + 2 * kStIRowFloats * 4);
                if (!MIXED) {
                    f2x2 old[4];
                    ring_wait_st();
                    ring_ld(t & 7, old);
                    ring_wait_ld();
                    ring_st(t & 7, av);
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
#pragma unroll
                        for (int j = 0; j < 4; ++j)
                            S2[MIXED ? 0 : q][j] = __dsub_rn(__dadd_rn(S2[MIXED ? 0 : q][j], w2(get(av[q], j), SLOW)), w2(get(old[q], j), SLOW));
                    }
                    emit(ro_y, o0, o1, o2);
                } else {
                    f2x2 pa[4], pb[4], pc[4], pd[4];
                    ring_wait_st();
                    ring_ld((t - 6) & 7, pa);
                    ring_ld((t - 4) & 7, pb);
                    ring_wait_ld();
#pragma unroll
                    for (int q = 0; q < 4; ++q) pa[q] = addp(pa[q], pb[q]);
                    ring_ld((t - 2) & 7, pc);
                    ring_ld(t & 7, pd);
                    ring_wait_ld();
#pragma unroll
                    for (int q = 0; q < 4; ++q) pd[q] = xadd(av[q], pd[q]);
                    ring_st(t & 7, pd);
                    ring_st((t + 1) & 7, av);
#pragma unroll
                    for (int q = 0; q < 4; ++q) pc[q] = addp(pc[q], pd[q]);
                    emit_pairs(ro_y, pa, pc, o0, o1, o2);
                }
                ro_y += rowB;
                __syncwarp();
                if (lane == 0) mbar_arrive(bar_empty + 8 * (k & (kStCoefStages - 1)));   // this warp is done with stage k
            };
            if (IW) {
                for (; t <= Ts1 && !slow; ++t) {
                    if (needs_slow(xn.p, xo.p)) { slow = true; break; }
                    steady_st(std::false_type{});
                }
            }
            for (; t <= Ts1; ++t) steady_st(std::true_type{});
        }
    }
    for (; t <= Tend; ++t) generic_step(t);
}

}  // namespace psm
