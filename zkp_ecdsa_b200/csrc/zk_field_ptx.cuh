// zk_field_ptx.cuh — sm_90a multiplier kernels for the two hot fields (device only).
//
// Measured on an H100 SXM 80GB at a 400 W power limit (tools/imad_peak.cu): IMAD.WIDE.U32 (32x32+64)
// issues at 31 /clk/SM — half the rate of a 32-bit IMAD — while IADD3 runs at ~110 /clk/SM on the
// other pipe and dual-issues with it.  So the cost of a modular multiplication is its number of 32x32 products; carries,
// shifts and small-constant multiples are free as long as they stay on the ALU pipe.
//
// Both routines are "finely integrated product scanning" (FIPS) Montgomery multiplications:
// column k accumulates sum a_i b_{k-i} + sum m_i p_{k-i} in a 96-bit register triple.  Each
// product is `mad.lo.cc / madc.hi.cc / addc`, which ptxas fuses into ONE IMAD.WIDE.U32 with
// carry-out plus one IADD3.X (checked with cuobjdump).
//
//  * tom.p  (9 limbs, lazy): p = [p0 p1 p2 p3 | 2 | 0 | 4 | 0xfffffffc | 3]; the quotient
//    digit m_i meets only five generic limbs (p0..p3, p7); 2m, 4m, 3m are shifts/adds.
//    81 + 45 = 126 products instead of 171.
//  * p256.p (8 limbs, strict): p = 2^256 - 2^224 + 2^192 + 2^96 - 1 and -1/p = 1 mod 2^32, so
//    m_i = column word and m_i*p is five signed word additions: column k gets
//    -m_k + m_{k-3} + m_{k-6} - m_{k-7} + m_{k-8}.  64 products instead of 136, no quotient mults.
//    Its squaring (p256_sqr_body) forms each cross product once: 36 products.
#pragma once
// included from zk_field.cuh after the field descriptors and multi-word helpers

#if defined(__CUDA_ARCH__)
namespace zk {
namespace ptx {

__device__ __forceinline__ void mac3(uint32_t& a0, uint32_t& a1, uint32_t& a2, uint32_t x, uint32_t y) {
  asm("mad.lo.cc.u32 %0, %3, %4, %0;\n\t"
      "madc.hi.cc.u32 %1, %3, %4, %1;\n\t"
      "addc.u32 %2, %2, 0;"
      : "+r"(a0), "+r"(a1), "+r"(a2)
      : "r"(x), "r"(y));
}
__device__ __forceinline__ void add3(uint32_t& a0, uint32_t& a1, uint32_t& a2, uint32_t lo, uint32_t hi) {
  asm("add.cc.u32 %0, %0, %3;\n\t"
      "addc.cc.u32 %1, %1, %4;\n\t"
      "addc.u32 %2, %2, 0;"
      : "+r"(a0), "+r"(a1), "+r"(a2)
      : "r"(lo), "r"(hi));
}
// signed 96-bit accumulator += / -= an unsigned word
__device__ __forceinline__ void addw(uint32_t& a0, uint32_t& a1, uint32_t& a2, uint32_t w) {
  asm("add.cc.u32 %0, %0, %3;\n\t"
      "addc.cc.u32 %1, %1, 0;\n\t"
      "addc.u32 %2, %2, 0;"
      : "+r"(a0), "+r"(a1), "+r"(a2)
      : "r"(w));
}
__device__ __forceinline__ void subw(uint32_t& a0, uint32_t& a1, uint32_t& a2, uint32_t w) {
  asm("sub.cc.u32 %0, %0, %3;\n\t"
      "subc.cc.u32 %1, %1, 0;\n\t"
      "subc.u32 %2, %2, 0;"
      : "+r"(a0), "+r"(a1), "+r"(a2)
      : "r"(w));
}

// x << n / x >> (32 - n) as funnel shifts: plain C shifts become IMAD.SHL / IMAD.U32 on the multiplier
// pipe (ptxas balances pipes assuming the FMA pipe is idle), which is the one pipe this code saturates.
__device__ __forceinline__ uint32_t shl_alu(uint32_t x, uint32_t n) {
  uint32_t r;
  asm("shf.l.clamp.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(0u), "r"(x), "r"(n));
  return r;
}
__device__ __forceinline__ uint32_t shr_top_alu(uint32_t x, uint32_t n) {   // x >> (32 - n)
  uint32_t r;
  asm("shf.l.clamp.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(x), "r"(0u), "r"(n));
  return r;
}

// r = a*b/2^288 mod tom.p, lazy: inputs < 2^13 p, output < 2p (no final subtraction).
__device__ __forceinline__ void tom_mul_body_ps(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = 9;
  constexpr uint32_t P0 = FpTom::p(0), P1 = FpTom::p(1), P2 = FpTom::p(2), P3 = FpTom::p(3), P7 = FpTom::p(7);
  static_assert(FpTom::p(4) == 2 && FpTom::p(5) == 0 && FpTom::p(6) == 4 && FpTom::p(8) == 3, "tom.p limb structure");
  uint32_t m[N], t[N];
  uint32_t a0 = 0, a1 = 0, a2 = 0;
  // (two accumulator triples per column for more ILP made the commit kernels slower and only single-thread
  //  chains faster — kept single)
#pragma unroll
  for (int k = 0; k < 2 * N; k++) {
    // a_i * b_{k-i}
#pragma unroll
    for (int i = 0; i < N; i++) {
      const int j = k - i;
      if (j >= 0 && j < N) mac3(a0, a1, a2, a[i], b[j]);
    }
    // m_i * p_{k-i}, i < min(k, N)   (p_j generic for j in {1,2,3,7}; shifts for j in {4,6,8})
#pragma unroll
    for (int i = 0; i < N; i++) {
      const int j = k - i;
      if (i < k && j >= 1 && j < N) {
        if (j == 1) mac3(a0, a1, a2, m[i], P1);
        else if (j == 2) mac3(a0, a1, a2, m[i], P2);
        else if (j == 3) mac3(a0, a1, a2, m[i], P3);
        else if (j == 7) mac3(a0, a1, a2, m[i], P7);
        else if (j == 4) add3(a0, a1, a2, shl_alu(m[i], 1), shr_top_alu(m[i], 1));
        else if (j == 6) add3(a0, a1, a2, shl_alu(m[i], 2), shr_top_alu(m[i], 2));
        else if (j == 8) { add3(a0, a1, a2, shl_alu(m[i], 1), shr_top_alu(m[i], 1)); add3(a0, a1, a2, m[i], 0u); }
      }
    }
    if (k < N) {
      m[k] = a0 * FpTom::kN0Inv;
      mac3(a0, a1, a2, m[k], P0);   // a0 becomes 0
    } else {
      t[k - N] = a0;
    }
    a0 = a1; a1 = a2; a2 = 0;
  }
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = t[i];
}

// ---------------------------------------------------------------------------------------------
// tom.p, operand scanning with even/odd accumulator arrays (the layout sppark / CGBN-style code uses).
// In product scanning every product goes through one 96-bit column accumulator, so each MAC reads the
// registers the previous MAC wrote; here each row is two carry chains of mad.lo.cc/madc.hi.cc pairs over
// DISTINCT accumulators and only the carry flag links consecutive instructions.  tools/mul_peak.cu (this
// multiplier alone, registers only): 0.67 -> 0.77 of the IMAD.WIDE peak at the commit kernels' occupancy.
//
// T = E + O: E holds 64-bit lanes at even limb positions (0,1),(2,3).., O at odd positions (1,2),(3,4)..
// Row i adds a_i*b (5 lanes into the array whose lanes start at position i, 4 into the other one), then
// m_i*p: generic limbs p0..p3 as MACs, 2, 4, 3 and 0xfffffffc = 2^32 - 4 as shifted adds inside the same
// carry chains.  The "stray" high half of the other array's lane (i-1, i) is folded into position i
// first, its carry enters the chain that starts at position i+1.
// 9 x (9 + 4) = 117 IMAD.WIDE per product.
template <int I, bool kFirst>
__device__ __forceinline__ void tom_row(uint32_t* A, uint32_t* Bq, uint32_t x, const uint32_t* b) {
  // chain 1: stray + a_i * b_{1,3,5,7} into Bq lanes (I+1,I+2) .. (I+7,I+8), carry into Bq[I+9]
  if (kFirst) {
    asm("mad.lo.cc.u32 %0, %9, %10, %0;\n\t"
        "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %11, %2;\n\t"
        "madc.hi.cc.u32 %3, %9, %11, %3;\n\t"
        "madc.lo.cc.u32 %4, %9, %12, %4;\n\t"
        "madc.hi.cc.u32 %5, %9, %12, %5;\n\t"
        "madc.lo.cc.u32 %6, %9, %13, %6;\n\t"
        "madc.hi.cc.u32 %7, %9, %13, %7;\n\t"
        "addc.u32 %8, %8, 0;"
        : "+r"(Bq[I + 1]), "+r"(Bq[I + 2]), "+r"(Bq[I + 3]), "+r"(Bq[I + 4]), "+r"(Bq[I + 5]), "+r"(Bq[I + 6]),
          "+r"(Bq[I + 7]), "+r"(Bq[I + 8]), "+r"(Bq[I + 9])
        : "r"(x), "r"(b[1]), "r"(b[3]), "r"(b[5]), "r"(b[7]));
  } else {
    asm("add.cc.u32 %0, %0, %10;\n\t"
        "madc.lo.cc.u32 %1, %11, %12, %1;\n\t"
        "madc.hi.cc.u32 %2, %11, %12, %2;\n\t"
        "madc.lo.cc.u32 %3, %11, %13, %3;\n\t"
        "madc.hi.cc.u32 %4, %11, %13, %4;\n\t"
        "madc.lo.cc.u32 %5, %11, %14, %5;\n\t"
        "madc.hi.cc.u32 %6, %11, %14, %6;\n\t"
        "madc.lo.cc.u32 %7, %11, %15, %7;\n\t"
        "madc.hi.cc.u32 %8, %11, %15, %8;\n\t"
        "addc.u32 %9, %9, 0;"
        : "+r"(A[I]), "+r"(Bq[I + 1]), "+r"(Bq[I + 2]), "+r"(Bq[I + 3]), "+r"(Bq[I + 4]), "+r"(Bq[I + 5]),
          "+r"(Bq[I + 6]), "+r"(Bq[I + 7]), "+r"(Bq[I + 8]), "+r"(Bq[I + 9])
        : "r"(Bq[I]), "r"(x), "r"(b[1]), "r"(b[3]), "r"(b[5]), "r"(b[7]));
  }
  // chain 2: a_i * b_{0,2,4,6,8} into A lanes (I,I+1) .. (I+8,I+9).  The top lane cannot carry out: it
  // holds a few carries of earlier rows, a_i*b_8 < 2^47 (b_8 < 2^15 for lazy operands < 2^13 p) and 3m.
  asm("mad.lo.cc.u32 %0, %11, %12, %0;\n\t"
      "madc.hi.cc.u32 %1, %11, %12, %1;\n\t"
      "madc.lo.cc.u32 %2, %11, %13, %2;\n\t"
      "madc.hi.cc.u32 %3, %11, %13, %3;\n\t"
      "madc.lo.cc.u32 %4, %11, %14, %4;\n\t"
      "madc.hi.cc.u32 %5, %11, %14, %5;\n\t"
      "madc.lo.cc.u32 %6, %11, %15, %6;\n\t"
      "madc.hi.cc.u32 %7, %11, %15, %7;\n\t"
      "madc.lo.cc.u32 %8, %11, %16, %8;\n\t"
      "madc.hi.u32 %9, %11, %16, %9;"
      : "+r"(A[I]), "+r"(A[I + 1]), "+r"(A[I + 2]), "+r"(A[I + 3]), "+r"(A[I + 4]), "+r"(A[I + 5]), "+r"(A[I + 6]),
        "+r"(A[I + 7]), "+r"(A[I + 8]), "+r"(A[I + 9]), "+r"(A[I + 10])
      : "r"(x), "r"(b[0]), "r"(b[2]), "r"(b[4]), "r"(b[6]), "r"(b[8]));
  // quotient digit and the small multiples of it
  const uint32_t m = A[I] * FpTom::kN0Inv;
  const uint32_t s1 = shl_alu(m, 1), t1 = shr_top_alu(m, 1), s2 = shl_alu(m, 2), t2 = shr_top_alu(m, 2);
  uint32_t lo3, hi3, lo7, hi7;
  asm("add.cc.u32 %0, %2, %3;\n\taddc.u32 %1, %4, 0;" : "=r"(lo3), "=r"(hi3) : "r"(s1), "r"(m), "r"(t1));      // 3m
  asm("sub.cc.u32 %0, 0, %2;\n\tsubc.u32 %1, %3, %4;" : "=r"(lo7), "=r"(hi7) : "r"(s2), "r"(m), "r"(t2));     // (2^32-4)m
  // chain 3: m * (p0, p2, 2, 4, 3) into the A lanes; A[I] becomes 0
  constexpr uint32_t P0 = FpTom::p(0), P1 = FpTom::p(1), P2 = FpTom::p(2), P3 = FpTom::p(3);
  asm("mad.lo.cc.u32 %0, %11, %12, %0;\n\t"
      "madc.hi.cc.u32 %1, %11, %12, %1;\n\t"
      "madc.lo.cc.u32 %2, %11, %13, %2;\n\t"
      "madc.hi.cc.u32 %3, %11, %13, %3;\n\t"
      "addc.cc.u32 %4, %4, %14;\n\t"
      "addc.cc.u32 %5, %5, %15;\n\t"
      "addc.cc.u32 %6, %6, %16;\n\t"
      "addc.cc.u32 %7, %7, %17;\n\t"
      "addc.cc.u32 %8, %8, %18;\n\t"
      "addc.u32 %9, %9, %19;"
      : "+r"(A[I]), "+r"(A[I + 1]), "+r"(A[I + 2]), "+r"(A[I + 3]), "+r"(A[I + 4]), "+r"(A[I + 5]), "+r"(A[I + 6]),
        "+r"(A[I + 7]), "+r"(A[I + 8]), "+r"(A[I + 9]), "+r"(A[I + 10])
      : "r"(m), "r"(P0), "r"(P2), "r"(s1), "r"(t1), "r"(s2), "r"(t2), "r"(lo3), "r"(hi3));
  // chain 4: m * (p1, p3, 0, 2^32-4) into the Bq lanes
  asm("mad.lo.cc.u32 %0, %9, %10, %0;\n\t"
      "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
      "madc.lo.cc.u32 %2, %9, %11, %2;\n\t"
      "madc.hi.cc.u32 %3, %9, %11, %3;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\t"
      "addc.cc.u32 %5, %5, 0;\n\t"
      "addc.cc.u32 %6, %6, %12;\n\t"
      "addc.cc.u32 %7, %7, %13;\n\t"
      "addc.u32 %8, %8, 0;"
      : "+r"(Bq[I + 1]), "+r"(Bq[I + 2]), "+r"(Bq[I + 3]), "+r"(Bq[I + 4]), "+r"(Bq[I + 5]), "+r"(Bq[I + 6]),
        "+r"(Bq[I + 7]), "+r"(Bq[I + 8]), "+r"(Bq[I + 9])
      : "r"(m), "r"(P1), "r"(P3), "r"(lo7), "r"(hi7));
}
// r = a*b/2^288 mod tom.p, lazy: inputs < 2^13 p, output < 2p (no final subtraction).
__device__ __forceinline__ void tom_mul_body(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  static_assert(FpTom::p(4) == 2 && FpTom::p(5) == 0 && FpTom::p(6) == 4 && FpTom::p(7) == 0xfffffffcu && FpTom::p(8) == 3,
                "tom.p limb structure");
  uint32_t E[20], O[20];
#pragma unroll
  for (int i = 0; i < 20; i++) { E[i] = 0; O[i] = 0; }
  tom_row<0, true>(E, O, a[0], b);
  tom_row<1, false>(O, E, a[1], b);
  tom_row<2, false>(E, O, a[2], b);
  tom_row<3, false>(O, E, a[3], b);
  tom_row<4, false>(E, O, a[4], b);
  tom_row<5, false>(O, E, a[5], b);
  tom_row<6, false>(E, O, a[6], b);
  tom_row<7, false>(O, E, a[7], b);
  tom_row<8, false>(E, O, a[8], b);
  // T / 2^288 = limbs 9..17 of E + O
  asm("add.cc.u32 %0, %9, %18;\n\t"
      "addc.cc.u32 %1, %10, %19;\n\t"
      "addc.cc.u32 %2, %11, %20;\n\t"
      "addc.cc.u32 %3, %12, %21;\n\t"
      "addc.cc.u32 %4, %13, %22;\n\t"
      "addc.cc.u32 %5, %14, %23;\n\t"
      "addc.cc.u32 %6, %15, %24;\n\t"
      "addc.cc.u32 %7, %16, %25;\n\t"
      "addc.u32 %8, %17, %26;"
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]), "=r"(r[8])
      : "r"(E[9]), "r"(E[10]), "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]), "r"(E[15]), "r"(E[16]), "r"(E[17]),
        "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]), "r"(O[15]), "r"(O[16]), "r"(O[17]));
}

// r = a*b/2^256 mod p256.p, strict: inputs < p, output < p.
// (product scanning: for this modulus it ran faster than the operand-scanning variant below, in tools/mul_peak
//  and in PhaseAP256Task, so it is the one in use.)
__device__ __forceinline__ void p256_mul_body(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = 8;
  uint32_t m[N], t[N + 1];
  uint32_t a0 = 0, a1 = 0, a2 = 0;   // signed 96-bit column accumulator (two's complement)
#pragma unroll
  for (int k = 0; k < 2 * N; k++) {
#pragma unroll
    for (int i = 0; i < N; i++) {
      const int j = k - i;
      if (j >= 0 && j < N) mac3(a0, a1, a2, a[i], b[j]);
    }
    // + m_{k-3} + m_{k-6} - m_{k-7} + m_{k-8}
    if (k - 3 >= 0 && k - 3 < N) addw(a0, a1, a2, m[k - 3 < 0 ? 0 : (k - 3 >= N ? 0 : k - 3)]);
    if (k - 6 >= 0 && k - 6 < N) addw(a0, a1, a2, m[k - 6 < 0 ? 0 : (k - 6 >= N ? 0 : k - 6)]);
    if (k - 7 >= 0 && k - 7 < N) subw(a0, a1, a2, m[k - 7 < 0 ? 0 : (k - 7 >= N ? 0 : k - 7)]);
    if (k - 8 >= 0 && k - 8 < N) addw(a0, a1, a2, m[k - 8 < 0 ? 0 : (k - 8 >= N ? 0 : k - 8)]);
    if (k < N) {
      m[k] = a0;          // -1/p = 1 mod 2^32: the quotient digit is the column word itself
      a0 = 0;             // column - m_k*1 clears the low word exactly (no borrow: a0 - a0)
    } else {
      t[k - N] = a0;
    }
    a0 = a1; a1 = a2; a2 = (uint32_t)((int32_t)a2 >> 31);
  }
  t[N] = a0;   // 0 or 1
  uint32_t u[N];
  uint32_t br = sub_p<FpP256>(u, t);
  const bool ge = (t[N] != 0) || (br == 0);
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = ge ? u[i] : t[i];
}

// r = a^2/2^256 mod p256.p, strict: input < p, output < p.  The columns of p256_mul_body with b = a: the cross
// products a_i a_j (i < j) of a column go into a triple of their own, which is doubled (three ALU additions) and
// added to the column accumulator with the square a_{k/2}^2 — the accumulator's carry-in must not be doubled.
// 28 + 8 = 36 products instead of 64; the reduction is the same additions-only one.
__device__ __forceinline__ void p256_sqr_body(uint32_t* r, const uint32_t* a) {
  constexpr int N = 8;
  uint32_t m[N], t[N + 1];
  uint32_t a0 = 0, a1 = 0, a2 = 0;   // signed 96-bit column accumulator (two's complement)
#pragma unroll
  for (int k = 0; k < 2 * N; k++) {
    if (k >= 1 && k <= 2 * N - 3) {  // columns with at least one cross product: 4 a_i a_j < 2^66, doubled < 2^67
      uint32_t c0 = 0, c1 = 0, c2 = 0;
#pragma unroll
      for (int i = 0; i < N; i++) {
        const int j = k - i;
        if (i < j && j < N) mac3(c0, c1, c2, a[i], a[j]);
      }
      asm("add.cc.u32 %0, %0, %0;\n\t"
          "addc.cc.u32 %1, %1, %1;\n\t"
          "addc.u32 %2, %2, %2;\n\t"
          "add.cc.u32 %3, %3, %0;\n\t"
          "addc.cc.u32 %4, %4, %1;\n\t"
          "addc.u32 %5, %5, %2;"
          : "+r"(c0), "+r"(c1), "+r"(c2), "+r"(a0), "+r"(a1), "+r"(a2));
    }
    if ((k & 1) == 0 && k / 2 < N) mac3(a0, a1, a2, a[k / 2], a[k / 2]);
    // + m_{k-3} + m_{k-6} - m_{k-7} + m_{k-8}
    if (k - 3 >= 0 && k - 3 < N) addw(a0, a1, a2, m[k - 3 < 0 ? 0 : (k - 3 >= N ? 0 : k - 3)]);
    if (k - 6 >= 0 && k - 6 < N) addw(a0, a1, a2, m[k - 6 < 0 ? 0 : (k - 6 >= N ? 0 : k - 6)]);
    if (k - 7 >= 0 && k - 7 < N) subw(a0, a1, a2, m[k - 7 < 0 ? 0 : (k - 7 >= N ? 0 : k - 7)]);
    if (k - 8 >= 0 && k - 8 < N) addw(a0, a1, a2, m[k - 8 < 0 ? 0 : (k - 8 >= N ? 0 : k - 8)]);
    if (k < N) {
      m[k] = a0;
      a0 = 0;
    } else {
      t[k - N] = a0;
    }
    a0 = a1; a1 = a2; a2 = (uint32_t)((int32_t)a2 >> 31);
  }
  t[N] = a0;   // 0 or 1
  uint32_t u[N];
  uint32_t br = sub_p<FpP256>(u, t);
  const bool ge = (t[N] != 0) || (br == 0);
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = ge ? u[i] : t[i];
}

// ---------------------------------------------------------------------------------------------
// p256.p, operand scanning with even/odd accumulator arrays (see tom_row).  -1/p = 1 mod 2^32, so the
// quotient digit of row i is the limb at position i itself, and m*p = m*(2^256 - 2^224 + 2^192 + 2^96 - 1)
// is the clearing of that limb plus ONE carry chain of plain additions on the same array:
//   +m at i+3, and m*(2^64 - 2^32 + 1) = (m, -m mod 2^32, m - [m != 0]) at i+6 .. i+8.
// 8 x 8 = 64 IMAD.WIDE per product.
template <int I, bool kFirst>
__device__ __forceinline__ void p256_row(uint32_t* A, uint32_t* Bq, uint32_t x, const uint32_t* b) {
  if (kFirst) {
    asm("mad.lo.cc.u32 %0, %9, %10, %0;\n\t"
        "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
        "madc.lo.cc.u32 %2, %9, %11, %2;\n\t"
        "madc.hi.cc.u32 %3, %9, %11, %3;\n\t"
        "madc.lo.cc.u32 %4, %9, %12, %4;\n\t"
        "madc.hi.cc.u32 %5, %9, %12, %5;\n\t"
        "madc.lo.cc.u32 %6, %9, %13, %6;\n\t"
        "madc.hi.cc.u32 %7, %9, %13, %7;\n\t"
        "addc.u32 %8, %8, 0;"
        : "+r"(Bq[I + 1]), "+r"(Bq[I + 2]), "+r"(Bq[I + 3]), "+r"(Bq[I + 4]), "+r"(Bq[I + 5]), "+r"(Bq[I + 6]),
          "+r"(Bq[I + 7]), "+r"(Bq[I + 8]), "+r"(Bq[I + 9])
        : "r"(x), "r"(b[1]), "r"(b[3]), "r"(b[5]), "r"(b[7]));
  } else {
    asm("add.cc.u32 %0, %0, %10;\n\t"
        "madc.lo.cc.u32 %1, %11, %12, %1;\n\t"
        "madc.hi.cc.u32 %2, %11, %12, %2;\n\t"
        "madc.lo.cc.u32 %3, %11, %13, %3;\n\t"
        "madc.hi.cc.u32 %4, %11, %13, %4;\n\t"
        "madc.lo.cc.u32 %5, %11, %14, %5;\n\t"
        "madc.hi.cc.u32 %6, %11, %14, %6;\n\t"
        "madc.lo.cc.u32 %7, %11, %15, %7;\n\t"
        "madc.hi.cc.u32 %8, %11, %15, %8;\n\t"
        "addc.u32 %9, %9, 0;"
        : "+r"(A[I]), "+r"(Bq[I + 1]), "+r"(Bq[I + 2]), "+r"(Bq[I + 3]), "+r"(Bq[I + 4]), "+r"(Bq[I + 5]),
          "+r"(Bq[I + 6]), "+r"(Bq[I + 7]), "+r"(Bq[I + 8]), "+r"(Bq[I + 9])
        : "r"(Bq[I]), "r"(x), "r"(b[1]), "r"(b[3]), "r"(b[5]), "r"(b[7]));
  }
  asm("mad.lo.cc.u32 %0, %9, %10, %0;\n\t"
      "madc.hi.cc.u32 %1, %9, %10, %1;\n\t"
      "madc.lo.cc.u32 %2, %9, %11, %2;\n\t"
      "madc.hi.cc.u32 %3, %9, %11, %3;\n\t"
      "madc.lo.cc.u32 %4, %9, %12, %4;\n\t"
      "madc.hi.cc.u32 %5, %9, %12, %5;\n\t"
      "madc.lo.cc.u32 %6, %9, %13, %6;\n\t"
      "madc.hi.cc.u32 %7, %9, %13, %7;\n\t"
      "addc.u32 %8, %8, 0;"
      : "+r"(A[I]), "+r"(A[I + 1]), "+r"(A[I + 2]), "+r"(A[I + 3]), "+r"(A[I + 4]), "+r"(A[I + 5]), "+r"(A[I + 6]),
        "+r"(A[I + 7]), "+r"(A[I + 8])
      : "r"(x), "r"(b[0]), "r"(b[2]), "r"(b[4]), "r"(b[6]));
  const uint32_t m = A[I];   // limb i is cleared by -m (never read again)
  uint32_t negm, third;
  asm("sub.cc.u32 %0, 0, %2;\n\tsubc.u32 %1, %2, 0;" : "=r"(negm), "=r"(third) : "r"(m));
  asm("add.cc.u32 %0, %0, %7;\n\t"
      "addc.cc.u32 %1, %1, 0;\n\t"
      "addc.cc.u32 %2, %2, 0;\n\t"
      "addc.cc.u32 %3, %3, %7;\n\t"
      "addc.cc.u32 %4, %4, %8;\n\t"
      "addc.cc.u32 %5, %5, %9;\n\t"
      "addc.u32 %6, %6, 0;"
      : "+r"(A[I + 3]), "+r"(A[I + 4]), "+r"(A[I + 5]), "+r"(A[I + 6]), "+r"(A[I + 7]), "+r"(A[I + 8]), "+r"(A[I + 9])
      : "r"(m), "r"(negm), "r"(third));
}
// operand-scanning variant (measured slower for p256.p, not used; bit-exact, GPU parity suite passed with it)
__device__ __forceinline__ void p256_mul_body_os(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  constexpr int N = 8;
  uint32_t E[18], O[18];
#pragma unroll
  for (int i = 0; i < 18; i++) { E[i] = 0; O[i] = 0; }
  p256_row<0, true>(E, O, a[0], b);
  p256_row<1, false>(O, E, a[1], b);
  p256_row<2, false>(E, O, a[2], b);
  p256_row<3, false>(O, E, a[3], b);
  p256_row<4, false>(E, O, a[4], b);
  p256_row<5, false>(O, E, a[5], b);
  p256_row<6, false>(E, O, a[6], b);
  p256_row<7, false>(O, E, a[7], b);
  uint32_t t[N + 1];
  asm("add.cc.u32 %0, %9, %18;\n\t"
      "addc.cc.u32 %1, %10, %19;\n\t"
      "addc.cc.u32 %2, %11, %20;\n\t"
      "addc.cc.u32 %3, %12, %21;\n\t"
      "addc.cc.u32 %4, %13, %22;\n\t"
      "addc.cc.u32 %5, %14, %23;\n\t"
      "addc.cc.u32 %6, %15, %24;\n\t"
      "addc.cc.u32 %7, %16, %25;\n\t"
      "addc.u32 %8, %17, %26;"
      : "=r"(t[0]), "=r"(t[1]), "=r"(t[2]), "=r"(t[3]), "=r"(t[4]), "=r"(t[5]), "=r"(t[6]), "=r"(t[7]), "=r"(t[8])
      : "r"(E[8]), "r"(E[9]), "r"(E[10]), "r"(E[11]), "r"(E[12]), "r"(E[13]), "r"(E[14]), "r"(E[15]), "r"(E[16]),
        "r"(O[8]), "r"(O[9]), "r"(O[10]), "r"(O[11]), "r"(O[12]), "r"(O[13]), "r"(O[14]), "r"(O[15]), "r"(O[16]));
  uint32_t u[N];
  uint32_t br = sub_p<FpP256>(u, t);
  const bool ge = (t[N] != 0) || (br == 0);
#pragma unroll
  for (int i = 0; i < N; i++) r[i] = ge ? u[i] : t[i];
}

// The multipliers are real (non-inlined) functions: operands and result travel in registers
// (by-value structs; the device ABI keeps them in R4..), and every warp of the SM executes the
// same ~5 KB body.  Fully inlining them made the commitment kernel ~130 KB of straight-line
// code and the warps stalled on instruction fetch.
struct V9 { uint32_t v[9]; };
struct V8 { uint32_t v[8]; };
static __device__ __noinline__ V9 tom_mul_fn(V9 a, V9 b) {
  V9 r;
  tom_mul_body(r.v, a.v, b.v);
  return r;
}
static __device__ __noinline__ V8 p256_mul_fn(V8 a, V8 b) {
  V8 r;
  p256_mul_body(r.v, a.v, b.v);
  return r;
}
static __device__ __noinline__ V8 p256_sqr_fn(V8 a) {
  V8 r;
  p256_sqr_body(r.v, a.v);
  return r;
}
__device__ __forceinline__ void tom_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
#if defined(ZKA_INLINE_MUL)
  tom_mul_body(r, a, b);
#else
  V9 x, y;
#pragma unroll
  for (int i = 0; i < 9; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  V9 z = tom_mul_fn(x, y);
#pragma unroll
  for (int i = 0; i < 9; i++) r[i] = z.v[i];
#endif
}
__device__ __forceinline__ void p256_mul(uint32_t* r, const uint32_t* a, const uint32_t* b) {
#if defined(ZKA_INLINE_MUL)
  p256_mul_body(r, a, b);
#else
  V8 x, y;
#pragma unroll
  for (int i = 0; i < 8; i++) { x.v[i] = a[i]; y.v[i] = b[i]; }
  V8 z = p256_mul_fn(x, y);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
#endif
}
__device__ __forceinline__ void p256_sqr(uint32_t* r, const uint32_t* a) {
#if defined(ZKA_INLINE_MUL)
  p256_sqr_body(r, a);
#else
  V8 x;
#pragma unroll
  for (int i = 0; i < 8; i++) x.v[i] = a[i];
  V8 z = p256_sqr_fn(x);
#pragma unroll
  for (int i = 0; i < 8; i++) r[i] = z.v[i];
#endif
}

}  // namespace ptx
}  // namespace zk
#endif
