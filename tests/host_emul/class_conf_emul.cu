// CPU emulation harness for the class-map epilogues' running arg-max and softmax (csrc/conv_common.cuh: ClassArg):
// the channels of each position are taken and the partial results joined in the order each epilogue uses.
//   order 0: one thread, every channel in ascending order (conv_simt_kernel; epilogue_rows with 8-column rounds)
//   order 1: epilogue_rows with 32-column rounds: thread h of a row takes channels [c0 + 16 h, c0 + 16 h + 16) of
//            every round c0, then the two threads join (class_arg_merge_xor(ca, 1))
//   order 2: epilogue_xp: lane q takes the 8-channel block [c0 + 8 (q & 1), + 8) of every 16-channel chunk c0
//            (class_take8), then lanes q and q ^ 1 join
#include "conv_common.cuh"

extern "C" void occd_set_last_error(const char*) {}

extern "C" int class_conf_emulate(const float* x, long long n_pos, int C, int order, int conf, unsigned short* cls,
                                  unsigned short* conf_bits) {
  if (C < 1 || C > 65535 || order < 0 || order > 2) return 1;
  const int N = (C + 15) / 16 * 16;   // the N tile of a class map covers Cout_pad
  for (long long p = 0; p < n_pos; ++p) {
    const float* v = x + p * C;
    ClassArg a = class_arg_init();
    if (order == 0) {
      for (int c = 0; c < C; ++c) class_arg_take(a, v[c], c, conf != 0);
    } else {
      const int round = order == 1 ? 32 : 16, width = round / 2;
      ClassArg part[2] = {class_arg_init(), class_arg_init()};
      for (int c0 = 0; c0 < N; c0 += round)
        for (int h = 0; h < 2; ++h)
          for (int i = 0; i < width; ++i) {
            const int c = c0 + width * h + i;
            if (c < C) class_arg_take(part[h], v[c], c, conf != 0);
          }
      a = part[0];
      class_arg_join(a, part[1], conf != 0);
    }
    cls[p] = (unsigned short)a.c;
    if (conf) {
      const __half_raw h = __float2half_rn(class_arg_conf(a));
      conf_bits[p] = h.x;
    }
  }
  return 0;
}
