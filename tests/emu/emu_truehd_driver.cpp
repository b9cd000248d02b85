// CPU build of the TrueHD decoder: sushi_b200/csrc/sb_truehd.cuh compiled with g++, driven the way sb_truehd.cu drives
// it (tests/test_kernel_emulation_truehd.py).  Every byte position holding a major-sync pattern is tried as a candidate
// (k_truehd_sync), the host chain walks the AU lengths into restart segments, each segment is decoded from a fresh
// state (k_truehd_decode) and the segments' checks are joined.  The chain and the checks are the library's own
// functions.
#include <stdint.h>
#include <string.h>
#include <vector>

#include "sb_truehd.cuh"

extern "C" {

// Decode a stream whose blocks start at blocks[0..n_blocks) of buf (where[]: each block's file offset, for messages).
// pcm receives the frames (at most cap; NULL: count only).  With period > 0 nothing is stored: each segment is decoded
// into a scratch buffer and compared with expect[], the stream's PCM repeating every `period` frames, and
// *mismatch receives the number of differing samples.  Segments decode in parallel (OpenMP), each from its own state.
// Returns the frame count, or -1 with the message in msg; info[0..1] = channels, sample rate.
int64_t emu_truehd_decode(const uint8_t* buf, int64_t nbytes, const int64_t* blocks, const int64_t* where, int64_t n_blocks,
                          int16_t* pcm, int64_t cap, int32_t* info, char* msg, int msg_len, const int16_t* expect,
                          int64_t period, int64_t* mismatch) {
    auto where_off = [&](int64_t off) {
        int64_t i = 0;
        while (i < n_blocks && blocks[i] <= off) ++i;
        return i > 0 && where[i - 1] >= 0 ? where[i - 1] : off;
    };
    sbthd::Format f;
    char m[200];
    if (!sbthd::parse_format(buf, nbytes, n_blocks ? blocks[0] : 0, &f, m, sizeof(m))) {
        snprintf(msg, msg_len, m, (long long)where_off(n_blocks ? blocks[0] : 0));
        return -1;
    }
    info[0] = f.channels; info[1] = f.rate;
    std::vector<sbthd::Candidate> cand;
    for (int64_t i = 0; i + 36 <= nbytes; ++i)
        if (buf[i + 4] == 0xF8 && buf[i + 5] == 0x72 && buf[i + 6] == 0x6F && (buf[i + 7] & 0xFE) == 0xBA) {
            sbthd::Candidate c = sbthd::candidate(buf, nbytes, i, f);
            if (c.code != sbthd::kBadSyncCrc) cand.push_back(c);
        }
    std::vector<sbthd::Segment> segs;
    int64_t n_au = 0;
    if (!sbthd::chain(buf, nbytes, blocks, n_blocks, cand, where_off, segs, &n_au, msg, msg_len)) return -1;
    const int64_t fs = (int64_t)f.spa * f.channels;
    std::vector<int16_t> out(period > 0 ? 0 : (size_t)(n_au * fs + 1));
    std::vector<sbthd::SegStatus> st(segs.size());
    int64_t bad = 0;
#pragma omp parallel reduction(+ : bad)
    {
        sbthd::State* state = new sbthd::State();
        std::vector<int16_t> scratch;
#pragma omp for schedule(dynamic, 64)
        for (int64_t k = 0; k < (int64_t)segs.size(); ++k) {
            const sbthd::Segment& g = segs[(size_t)k];
            int16_t* dst = out.data() + (period > 0 ? 0 : g.first_au * fs);
            if (period > 0) { scratch.assign((size_t)(g.n_au * fs), 0); dst = scratch.data(); }
            st[(size_t)k] = sbthd::decode_segment(buf, nbytes, blocks, n_blocks, f, g, k == 0, *state, dst);
            if (period > 0)
                for (int64_t j = 0; j < g.n_au * f.spa; ++j)
                    for (int c = 0; c < f.channels; ++c)
                        bad += scratch[(size_t)(j * f.channels + c)] != expect[((g.first_au * f.spa + j) % period) * f.channels + c];
        }
        delete state;
    }
    // the AU offsets, for messages: walk the failing segment again
    auto where_au = [&](int64_t k, int64_t au) {
        int64_t off = segs[(size_t)k].offset;
        for (int64_t a = segs[(size_t)k].first_au; a < au; ++a) off += (int64_t)(((buf[off] << 8) | buf[off + 1]) & 0xFFF) * 2;
        return where_off(off);
    };
    const int64_t frames = sbthd::check_segments(segs, st.data(), f, where_au, msg, msg_len);
    if (frames < 0) return -1;
    if (mismatch) *mismatch = bad;
    if (pcm && period <= 0) memcpy(pcm, out.data(), sizeof(int16_t) * (size_t)std::min(frames, cap) * f.channels);
    return frames;
}

}  // extern "C"
