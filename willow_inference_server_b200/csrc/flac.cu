// FLAC stream decoder (host code, no device work): the ingest format of the reference's fixtures and of /api/asr
// uploads.  The reference decodes with librosa/soundfile (main.py:579 `librosa.load(audio_file,
// sr=16000)`; fixtures client/{3sec,10sec,30sec}.flac); SURVEY.md section 8(f) row 3a asks for a decoder verified by the
// PCM MD5 every FLAC file carries in STREAMINFO.  Written from the FLAC format specification (frame / subframe /
// residual layout, CRC-8 0x07 on the frame header, CRC-16 0x8005 on the frame); integer exact.
//
// Supported: 4..32 bits per sample (decoded into int32), 1..8 channels, all subframe types (constant, verbatim, fixed
// 0-4, LPC 1-32), Rice / Rice2 partitions with escapes, wasted bits, the three stereo decorrelation modes, fixed and
// variable block size streams, metadata blocks skipped.  Not supported: Ogg encapsulation.
#include <stdint.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/wisb200.h"

namespace {

thread_local std::string g_flac_error;

struct FlacError {
  std::string msg;
};
[[noreturn]] void fail(const std::string& m) { throw FlacError{m}; }

struct BitReader {
  const uint8_t* p;
  size_t n;        // bytes
  size_t pos = 0;  // bit position
  BitReader(const uint8_t* d, size_t len) : p(d), n(len) {}
  size_t byte_pos() const { return pos >> 3; }
  bool aligned() const { return (pos & 7) == 0; }
  uint32_t bit() {
    if ((pos >> 3) >= n) fail("unexpected end of stream");
    const uint32_t v = (p[pos >> 3] >> (7 - (pos & 7))) & 1u;
    ++pos;
    return v;
  }
  uint64_t bits(int k) {  // k <= 57
    uint64_t v = 0;
    while (k > 0) {
      if ((pos >> 3) >= n) fail("unexpected end of stream");
      const int avail = 8 - static_cast<int>(pos & 7);
      const int take = k < avail ? k : avail;
      const uint32_t byte = p[pos >> 3];
      v = (v << take) | ((byte >> (avail - take)) & ((1u << take) - 1u));
      pos += take;
      k -= take;
    }
    return v;
  }
  int64_t sbits(int k) {
    if (k == 0) return 0;
    const uint64_t v = bits(k > 57 ? 57 : k);
    if (k > 57) fail("sample width not supported");
    const uint64_t sign = 1ull << (k - 1);
    return static_cast<int64_t>((v ^ sign)) - static_cast<int64_t>(sign);
  }
  uint32_t unary() {  // number of 0 bits before the next 1 bit
    uint32_t q = 0;
    for (;;) {
      if ((pos >> 3) >= n) fail("unexpected end of stream");
      // fast path: scan the rest of the current byte
      const int avail = 8 - static_cast<int>(pos & 7);
      const uint32_t rest = p[pos >> 3] & ((1u << avail) - 1u);
      if (rest == 0) {
        q += avail;
        pos += avail;
        continue;
      }
      int lead = 0;
      while (((rest >> (avail - 1 - lead)) & 1u) == 0) ++lead;
      q += lead;
      pos += lead + 1;
      return q;
    }
  }
  void align() { pos = (pos + 7) & ~static_cast<size_t>(7); }
};

uint8_t crc8(const uint8_t* d, size_t n) {
  uint8_t c = 0;
  for (size_t i = 0; i < n; ++i) {
    c ^= d[i];
    for (int b = 0; b < 8; ++b) c = static_cast<uint8_t>((c & 0x80) ? (c << 1) ^ 0x07 : (c << 1));
  }
  return c;
}
uint16_t crc16(const uint8_t* d, size_t n) {
  uint16_t c = 0;
  for (size_t i = 0; i < n; ++i) {
    c ^= static_cast<uint16_t>(d[i]) << 8;
    for (int b = 0; b < 8; ++b) c = static_cast<uint16_t>((c & 0x8000) ? (c << 1) ^ 0x8005 : (c << 1));
  }
  return c;
}

struct StreamInfo {
  int min_block = 0, max_block = 0, sample_rate = 0, channels = 0, bps = 0;
  uint64_t total = 0;
  uint8_t md5[16] = {0};
};

// "fLaC" + metadata blocks; returns the offset of the first frame
size_t parse_metadata(const uint8_t* d, size_t n, StreamInfo& si) {
  if (n < 42 || memcmp(d, "fLaC", 4) != 0) fail("not a FLAC stream (no fLaC marker)");
  size_t pos = 4;
  bool seen = false;
  for (;;) {
    if (pos + 4 > n) fail("truncated metadata");
    const bool last = (d[pos] & 0x80) != 0;
    const int type = d[pos] & 0x7F;
    const size_t len = (static_cast<size_t>(d[pos + 1]) << 16) | (static_cast<size_t>(d[pos + 2]) << 8) | d[pos + 3];
    pos += 4;
    if (pos + len > n) fail("truncated metadata block");
    if (type == 0) {
      if (len != 34) fail("bad STREAMINFO length");
      BitReader br(d + pos, len);
      si.min_block = static_cast<int>(br.bits(16));
      si.max_block = static_cast<int>(br.bits(16));
      br.bits(24);
      br.bits(24);
      si.sample_rate = static_cast<int>(br.bits(20));
      si.channels = static_cast<int>(br.bits(3)) + 1;
      si.bps = static_cast<int>(br.bits(5)) + 1;
      si.total = br.bits(36);
      memcpy(si.md5, d + pos + 18, 16);
      seen = true;
    } else if (type == 127) {
      fail("invalid metadata block type");
    }
    pos += len;
    if (last) break;
  }
  if (!seen) fail("no STREAMINFO block");
  if (si.sample_rate == 0 || si.bps < 4 || si.bps > 32) fail("unsupported STREAMINFO values");
  return pos;
}

void decode_residual(BitReader& br, int order, int blocksize, std::vector<int64_t>& out) {
  const int method = static_cast<int>(br.bits(2));
  if (method > 1) fail("reserved residual coding method");
  const int pbits = method == 0 ? 4 : 5;
  const uint32_t escape = method == 0 ? 15u : 31u;
  const int po = static_cast<int>(br.bits(4));
  const int parts = 1 << po;
  if ((blocksize >> po) << po != blocksize && po > 0) fail("block size not divisible by the partition count");
  int idx = order;
  for (int part = 0; part < parts; ++part) {
    int count = (po == 0) ? blocksize - order : (blocksize >> po) - (part == 0 ? order : 0);
    if (count < 0) fail("partition smaller than the predictor order");
    const uint32_t k = static_cast<uint32_t>(br.bits(pbits));
    if (k == escape) {
      const int raw = static_cast<int>(br.bits(5));
      for (int i = 0; i < count; ++i) out[idx++] = br.sbits(raw);
    } else {
      for (int i = 0; i < count; ++i) {
        const uint64_t q = br.unary();
        const uint64_t u = (q << k) | (k ? br.bits(static_cast<int>(k)) : 0);
        out[idx++] = static_cast<int64_t>(u >> 1) ^ -static_cast<int64_t>(u & 1);
      }
    }
  }
  if (idx != blocksize) fail("residual length mismatch");
}

void decode_subframe(BitReader& br, int bps, int blocksize, std::vector<int64_t>& s) {
  if (br.bit() != 0) fail("subframe padding bit set");
  const int type = static_cast<int>(br.bits(6));
  int wasted = 0;
  if (br.bit()) wasted = static_cast<int>(br.unary()) + 1;
  bps -= wasted;
  if (bps < 1) fail("wasted bits exceed the sample width");
  s.assign(blocksize, 0);
  if (type == 0) {  // constant
    const int64_t v = br.sbits(bps);
    for (int i = 0; i < blocksize; ++i) s[i] = v;
  } else if (type == 1) {  // verbatim
    for (int i = 0; i < blocksize; ++i) s[i] = br.sbits(bps);
  } else if (type >= 8 && type <= 12) {  // fixed predictor, order type - 8
    const int order = type - 8;
    if (order > blocksize) fail("predictor order exceeds the block size");
    for (int i = 0; i < order; ++i) s[i] = br.sbits(bps);
    decode_residual(br, order, blocksize, s);
    for (int i = order; i < blocksize; ++i) {
      int64_t pred = 0;
      switch (order) {
        case 1: pred = s[i - 1]; break;
        case 2: pred = 2 * s[i - 1] - s[i - 2]; break;
        case 3: pred = 3 * s[i - 1] - 3 * s[i - 2] + s[i - 3]; break;
        case 4: pred = 4 * s[i - 1] - 6 * s[i - 2] + 4 * s[i - 3] - s[i - 4]; break;
        default: break;
      }
      s[i] += pred;
    }
  } else if (type >= 32) {  // LPC, order (type & 31) + 1
    const int order = (type & 31) + 1;
    if (order > blocksize) fail("predictor order exceeds the block size");
    for (int i = 0; i < order; ++i) s[i] = br.sbits(bps);
    const int prec = static_cast<int>(br.bits(4)) + 1;
    if (prec == 16) fail("invalid LPC precision");
    const int shift = static_cast<int>(br.sbits(5));
    if (shift < 0) fail("negative LPC shift");
    int64_t coef[32];
    for (int j = 0; j < order; ++j) coef[j] = br.sbits(prec);
    decode_residual(br, order, blocksize, s);
    for (int i = order; i < blocksize; ++i) {
      int64_t acc = 0;
      for (int j = 0; j < order; ++j) acc += coef[j] * s[i - 1 - j];
      s[i] += acc >> shift;
    }
  } else {
    fail("reserved subframe type");
  }
  if (wasted)
    for (int i = 0; i < blocksize; ++i) s[i] = s[i] * (static_cast<int64_t>(1) << wasted);
}

uint64_t read_utf8_number(BitReader& br) {
  const uint32_t b0 = static_cast<uint32_t>(br.bits(8));
  int extra;
  uint64_t v;
  if (b0 < 0x80) return b0;
  if ((b0 & 0xE0) == 0xC0) { extra = 1; v = b0 & 0x1F; }
  else if ((b0 & 0xF0) == 0xE0) { extra = 2; v = b0 & 0x0F; }
  else if ((b0 & 0xF8) == 0xF0) { extra = 3; v = b0 & 0x07; }
  else if ((b0 & 0xFC) == 0xF8) { extra = 4; v = b0 & 0x03; }
  else if ((b0 & 0xFE) == 0xFC) { extra = 5; v = b0 & 0x01; }
  else if (b0 == 0xFE) { extra = 6; v = 0; }
  else fail("bad frame number coding");
  for (int i = 0; i < extra; ++i) {
    const uint32_t b = static_cast<uint32_t>(br.bits(8));
    if ((b & 0xC0) != 0x80) fail("bad frame number coding");
    v = (v << 6) | (b & 0x3F);
  }
  return v;
}

// decodes every frame; out = interleaved int32 samples (may be null: count only)
uint64_t decode_frames(const uint8_t* d, size_t n, size_t pos, const StreamInfo& si, int32_t* out, uint64_t cap_frames) {
  uint64_t done = 0;
  std::vector<std::vector<int64_t>> ch(si.channels);
  while (pos + 2 <= n && (si.total == 0 || done < si.total)) {
    BitReader br(d + pos, n - pos);
    if (br.bits(14) != 0x3FFE) fail("lost frame sync at byte " + std::to_string(pos));
    if (br.bit()) fail("reserved bit set in frame header");
    br.bit();  // blocking strategy (the coded number is then a sample number instead of a frame number)
    const int bs_code = static_cast<int>(br.bits(4));
    const int sr_code = static_cast<int>(br.bits(4));
    const int ca = static_cast<int>(br.bits(4));
    const int ss_code = static_cast<int>(br.bits(3));
    if (br.bit()) fail("reserved bit set in frame header");
    read_utf8_number(br);
    int blocksize;
    if (bs_code == 0) fail("reserved block size code");
    else if (bs_code == 1) blocksize = 192;
    else if (bs_code <= 5) blocksize = 576 << (bs_code - 2);
    else if (bs_code == 6) blocksize = static_cast<int>(br.bits(8)) + 1;
    else if (bs_code == 7) blocksize = static_cast<int>(br.bits(16)) + 1;
    else blocksize = 256 << (bs_code - 8);
    if (sr_code == 12) br.bits(8);
    else if (sr_code == 13 || sr_code == 14) br.bits(16);
    else if (sr_code == 15) fail("invalid sample rate code");
    const size_t hdr_bytes = br.byte_pos();
    const uint32_t c8 = static_cast<uint32_t>(br.bits(8));
    if (crc8(d + pos, hdr_bytes) != c8) fail("frame header CRC-8 mismatch");
    static const int ss_bits[8] = {0, 8, 12, -1, 16, 20, 24, 32};
    int bps = ss_bits[ss_code];
    if (bps < 0) fail("reserved sample size code");
    if (bps == 0) bps = si.bps;
    int nch;
    if (ca < 8) nch = ca + 1;
    else if (ca <= 10) nch = 2;
    else fail("reserved channel assignment");
    if (nch != si.channels) fail("channel count changes inside the stream");
    for (int c = 0; c < nch; ++c) {
      // the side channel of a decorrelated pair carries one extra bit
      const bool side = (ca == 8 && c == 1) || (ca == 9 && c == 0) || (ca == 10 && c == 1);
      decode_subframe(br, bps + (side ? 1 : 0), blocksize, ch[c]);
    }
    br.align();
    const size_t body = br.byte_pos();
    const uint32_t c16 = static_cast<uint32_t>(br.bits(16));
    if (crc16(d + pos, body) != c16) fail("frame CRC-16 mismatch");
    if (ca == 8) {  // left / side
      for (int i = 0; i < blocksize; ++i) ch[1][i] = ch[0][i] - ch[1][i];
    } else if (ca == 9) {  // side / right
      for (int i = 0; i < blocksize; ++i) ch[0][i] = ch[0][i] + ch[1][i];
    } else if (ca == 10) {  // mid / side
      for (int i = 0; i < blocksize; ++i) {
        const int64_t side = ch[1][i];
        const int64_t mid = (ch[0][i] * 2) | (side & 1);
        ch[0][i] = (mid + side) >> 1;
        ch[1][i] = (mid - side) >> 1;
      }
    }
    uint64_t keep = static_cast<uint64_t>(blocksize);
    if (si.total && done + keep > si.total) keep = si.total - done;
    if (out != nullptr) {
      if (done + keep > cap_frames) fail("output buffer too small");
      for (uint64_t i = 0; i < keep; ++i)
        for (int c = 0; c < nch; ++c) out[(done + i) * nch + c] = static_cast<int32_t>(ch[c][i]);
    }
    done += keep;
    pos += br.byte_pos();
  }
  if (si.total && done != si.total) fail("stream ends before the sample count announced in STREAMINFO");
  return done;
}

template <typename F>
int flac_guard(F&& f) {
  try {
    f();
    return 0;
  } catch (const FlacError& e) {
    g_flac_error = e.msg;
    return 1;
  } catch (const std::exception& e) {
    g_flac_error = e.what();
    return 2;
  }
}

}  // namespace

extern "C" {

const char* wisb_flac_last_error(void) { return g_flac_error.c_str(); }

int wisb_flac_info(const void* data, size_t nbytes, int32_t* sample_rate, int32_t* channels, int32_t* bits_per_sample,
                   int64_t* n_frames, uint8_t* md5_16) {
  return flac_guard([&] {
    if (data == nullptr) fail("data is NULL");
    StreamInfo si;
    const size_t first = parse_metadata(static_cast<const uint8_t*>(data), nbytes, si);
    uint64_t total = si.total;
    if (total == 0) total = decode_frames(static_cast<const uint8_t*>(data), nbytes, first, si, nullptr, 0);
    if (sample_rate) *sample_rate = si.sample_rate;
    if (channels) *channels = si.channels;
    if (bits_per_sample) *bits_per_sample = si.bps;
    if (n_frames) *n_frames = static_cast<int64_t>(total);
    if (md5_16) memcpy(md5_16, si.md5, 16);
  });
}

int wisb_flac_decode(const void* data, size_t nbytes, int32_t* out_interleaved, int64_t capacity_frames, int64_t* n_frames) {
  return flac_guard([&] {
    if (data == nullptr || out_interleaved == nullptr) fail("data / out is NULL");
    StreamInfo si;
    const size_t first = parse_metadata(static_cast<const uint8_t*>(data), nbytes, si);
    const uint64_t got = decode_frames(static_cast<const uint8_t*>(data), nbytes, first, si, out_interleaved,
                                       static_cast<uint64_t>(capacity_frames < 0 ? 0 : capacity_frames));
    if (n_frames) *n_frames = static_cast<int64_t>(got);
  });
}

}  // extern "C"
