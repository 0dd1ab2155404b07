// bz2enc_multi_emul.cpp -- TEST INFRASTRUCTURE: the device BZip2 encoder's multi-stream driver (bz2e::encode_streams) on
// the CPU emulation (cuda_emu.h).  Streams are laid out as b200z_bzip2_encode_batch lays out one device group: each
// starts on a 4 KiB input tile, in stream order.  Built by tests/test_bzip2_enc_batch_emul.py.
#define B200Z_EMU 1
#include "../../archive_b200/csrc/bzip2_enc_kernels.cu"


// Stream i is in_base[in_off[i] .. +in_len[i]).  out receives stream i at out_off[i] (set here: slots of
// bound(in_len) bytes, back to back; the caller gives sum of bound + 64 per stream), out_len[i] its length, crc32[i]
// its CRC-32.  max_batch 0: the built-in plan.  stats5: blocks, serially sorted blocks, rounds, 0, block batches.
extern "C" int emu_bzip2_encode_multi(const uint8_t *in_base, const uint64_t *in_off, const uint64_t *in_len, size_t n,
                                      uint32_t max_batch, uint8_t *out, uint64_t *out_off, uint64_t *out_len,
                                      uint32_t *crc32, uint32_t *stats5) {
  using namespace b200z::bz2e;
  std::vector<StreamDesc> sd(n);
  PlanSums sums;
  unsigned long long in0 = 0, out0 = 0;
  uint32_t blk0 = 0;
  for (size_t i = 0; i < n; ++i) {
    const size_t len = in_len[i];
    plan_add(sums, len);
    const unsigned long long cap = (bound(len) + 64 + 255) & ~255ull;
    sd[i] = StreamDesc{(uint32_t)in0, (uint32_t)len, (uint32_t)(in0 / 4096), tiles_of(len), blk0, max_blocks_of(len), out0, cap};
    in0 += (len + 4095) & ~4095ull;
    blk0 += sd[i].max_blocks;
    out0 += cap;
  }
  Plan p = plan_of(sums, (size_t)3 << 30);
  if (max_batch && max_batch < p.batch) p.batch = max_batch;
  uint8_t *staged = (uint8_t *)malloc(in0 + 64);
  memset(staged, 0xa5, in0 + 64);  // padding between streams: bytes no stream may read
  for (size_t i = 0; i < n; ++i) memcpy(staged + sd[i].in0, in_base + in_off[i], in_len[i]);
  void *ws = calloc(p.ws_bytes, 1);
  uint8_t *obuf = (uint8_t *)calloc(out0 + 16, 1);
  std::vector<unsigned long long> lens(n);
  std::vector<uint32_t> tile_crc(p.n_tiles);
  Stats st{0, 0, 0, 0, 0};
  int rc = encode_streams(staged, sd.data(), obuf, ws, p, lens.data(), tile_crc.data(), &st, nullptr);
  if (rc == 0) {
    unsigned long long at = 0;
    for (size_t i = 0; i < n; ++i) {
      out_off[i] = at;
      out_len[i] = lens[i];
      memcpy(out + at, obuf + sd[i].out0, lens[i]);
      at += lens[i];
      crc32[i] = crc32_fold(tile_crc.data() + sd[i].tile0, in_len[i]);
    }
  }
  if (stats5) memcpy(stats5, &st, 20);
  free(ws);
  free(obuf);
  free(staged);
  return rc;
}
