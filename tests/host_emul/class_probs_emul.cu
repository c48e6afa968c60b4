// CPU emulation harness for the class-map epilogues' probabilities (OCCD_OUT1_CLASS_U16_PROBS, csrc/conv_common.cuh):
// the running arg-max and softmax in each epilogue's merge order (the orders of class_conf_emul.cu), then the second
// pass that turns every channel's value into its probability with class_arg_prob.  Writes the class, the confidence
// bits of mode 4 and the probability bits [n_pos][C].
#include "conv_common.cuh"

extern "C" void occd_set_last_error(const char*) {}

extern "C" int class_probs_emulate(const float* x, long long n_pos, int C, int order, unsigned short* cls,
                                   unsigned short* conf_bits, unsigned short* prob_bits) {
  if (C < 1 || C > 65535 || order < 0 || order > 2) return 1;
  const int N = (C + 15) / 16 * 16;
  for (long long p = 0; p < n_pos; ++p) {
    const float* v = x + p * C;
    ClassArg a = class_arg_init();
    if (order == 0) {
      for (int c = 0; c < C; ++c) class_arg_take(a, v[c], c, true);
    } else {
      const int round = order == 1 ? 32 : 16, width = round / 2;
      ClassArg part[2] = {class_arg_init(), class_arg_init()};
      for (int c0 = 0; c0 < N; c0 += round)
        for (int h = 0; h < 2; ++h)
          for (int i = 0; i < width; ++i) {
            const int c = c0 + width * h + i;
            if (c < C) class_arg_take(part[h], v[c], c, true);
          }
      // class_arg_merge_xor: each lane joins the other's partial result into its own; both must agree
      ClassArg b = part[1];
      a = part[0];
      class_arg_join(a, part[1], true);
      class_arg_join(b, part[0], true);
      if (!(a.m == b.m || (a.m != a.m && b.m != b.m)) || !(a.s == b.s || (a.s != a.s && b.s != b.s)) || a.c != b.c)
        return 2;
    }
    cls[p] = (unsigned short)a.c;
    conf_bits[p] = __half_raw(__float2half_rn(class_arg_conf(a))).x;
    for (int c = 0; c < C; ++c) prob_bits[p * C + c] = __half_raw(__float2half_rn(class_arg_prob(a, v[c]))).x;
  }
  return 0;
}
