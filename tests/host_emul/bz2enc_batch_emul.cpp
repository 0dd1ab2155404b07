// bz2enc_batch_emul.cpp -- TEST INFRASTRUCTURE: the device BZip2 encoder on the CPU emulation (cuda_emu.h) with a cap on
// the blocks sorted and coded together, so that inputs of a few blocks run through several batches.  Built by
// tests/test_bzip2_enc_edges_emul.py.
#define B200Z_EMU 1
#include "../../archive_b200/csrc/bzip2_enc_kernels.cu"

// max_batch 0: the built-in plan.  stats4: n_blocks, n_serial_blocks, rounds, 0
extern "C" int emu_bzip2_encode_batch(const uint8_t *in, size_t n, uint8_t *out, size_t out_cap, size_t *out_len,
                                      uint32_t *stats4, uint32_t max_batch) {
  using namespace b200z::bz2e;
  Plan p = plan(n, (size_t)3 << 30);
  if (max_batch && max_batch < p.batch) p.batch = max_batch;
  void *ws = calloc(p.ws_bytes, 1);
  uint8_t *obuf = (uint8_t *)calloc(out_cap + 16, 1);
  Stats st{0, 0, 0, 0};
  int rc = encode_device(in, n, obuf, out_cap, ws, p, out_len, &st, nullptr);
  if (rc == 0) memcpy(out, obuf, *out_len);
  if (stats4) memcpy(stats4, &st, 16);
  free(ws);
  free(obuf);
  return rc;
}
