// The non-finite policy of the training losses, written once for csrc/losses.cu and csrc/iuv_train.cu.
//
//   smooth-L1 gradient   clamp(d, -1, 1), and NaN for a NaN difference, as torch's smooth_l1_loss backward gives
//                        (fminf / fmaxf alone return the other operand and would turn NaN into -1).
//   online log-sum-exp   running maximum m and sum s of exp(x - m) over a row of logits.  A -inf logit adds
//                        nothing: before the first finite logit m is still -inf and exp(-inf - -inf) would be NaN.
//                        A NaN or +inf logit makes s NaN, and a row of -inf only leaves m = -inf, s = 0; either way
//                        the row's loss and every gradient of it are NaN, as torch's cross_entropy gives.
// For finite inputs both do the floating-point operations the losses did before, in the same order.
#pragma once
#include <math.h>

namespace danet {

__host__ __device__ inline float sl1_grad(float d) { return d != d ? d : fminf(fmaxf(d, -1.f), 1.f); }

__host__ __device__ inline void lse_step(float x, float& m, float& s) {
    if (x > m) { s = x < INFINITY ? s * expf(m - x) + 1.f : NAN; m = x; }
    else if (x != -INFINITY) s += expf(x - m);
}

}  // namespace danet
