// grl_hd.h -- the one host/device qualifier and the correctly rounded operations of the closed forms that the host
// entries (grl_*_host) and the kernels both evaluate.
//
// Rule: every floating-point operation of a closed form shared by host and device goes through these, so both sides
// evaluate the same IEEE operations in the same order.  On the device each is the CUDA intrinsic, which nvcc never
// contracts into an FMA; on the host it is the plain operator (or libm sqrt / fma), and the host compiler runs with
// -ffp-contract=off (build.py), so it never contracts either.  Float and double take separate names, not overloads,
// so every call states the precision it rounds in.
#pragma once

#include <math.h>

#if defined(__CUDACC__)
#define GRL_HD __host__ __device__ __forceinline__
#else
#define GRL_HD inline
#endif

#if defined(__CUDA_ARCH__)
#define GRL_RN(dev, host) dev
#else
#define GRL_RN(dev, host) host
#endif

namespace grl {

GRL_HD float fadd_rn(float a, float b) { return GRL_RN(__fadd_rn(a, b), a + b); }
GRL_HD float fmul_rn(float a, float b) { return GRL_RN(__fmul_rn(a, b), a * b); }
GRL_HD float fdiv_rn(float a, float b) { return GRL_RN(__fdiv_rn(a, b), a / b); }

GRL_HD double dadd_rn(double a, double b) { return GRL_RN(__dadd_rn(a, b), a + b); }
GRL_HD double dsub_rn(double a, double b) { return GRL_RN(__dsub_rn(a, b), a - b); }
GRL_HD double dmul_rn(double a, double b) { return GRL_RN(__dmul_rn(a, b), a * b); }
GRL_HD double ddiv_rn(double a, double b) { return GRL_RN(__ddiv_rn(a, b), a / b); }
GRL_HD double dsqrt_rn(double a) { return GRL_RN(__dsqrt_rn(a), sqrt(a)); }
GRL_HD double dfma_rn(double a, double b, double c) { return GRL_RN(__fma_rn(a, b, c), fma(a, b, c)); }

}  // namespace grl

#undef GRL_RN
