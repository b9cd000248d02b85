// FLAC input: the file's frames decoded on the GPU into the interleaved int16 PCM that sb_load_pcm decodes from a WAV
// file, then the loader's own kernel (k_decode_resample_pad, width 2) from there on.
//   sb_flac_decode_file    upload the file; k_flac_sync lists every byte position holding a sync code and a frame
//                   header that parses, agrees with STREAMINFO and passes its CRC-8 (false syncs included); the host
//                   chains the real frames from the first one by their coded frame / sample numbers
//   sb_flac_decode_frames  the same for frames a container lists (Matroska blocks and laces): k_flac_frames, one
//                   thread per listed frame, checks the header at its offset; sample positions are the prefix sum of
//                   the block sizes, and errors name the file offset of the frame's block
//   then both       k_flac_decode: one thread per frame decodes its subframes in turn (a subframe starts where the
//                   previous one ends) and checks the frame's CRC-16 and end; k_flac_decorrelate: one CTA per frame
//                   undoes the stereo decorrelation and writes int16 (24-bit: the top 16 bits) into an sb_pcm
// The per-frame arithmetic is in sb_flac.cuh, shared with the CPU emulation of the tests.
#include "sb_decode.h"
#include "sb_flac.cuh"
#include <algorithm>
#include <vector>

using namespace sb;

namespace {

using sbflac::Candidate;
using sbflac::FrameDesc;

__global__ void __launch_bounds__(256)
k_flac_sync(const uint8_t* __restrict__ file, int64_t first, int64_t nbytes, int channels, int bits, int rate,
            Candidate* __restrict__ out, unsigned long long* __restrict__ count, int64_t cap) {
    const int64_t words = (nbytes + 3) >> 2;                       // the buffer is zero-padded past nbytes
    for (int64_t w = (first >> 2) + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < words;
         w += (int64_t)gridDim.x * blockDim.x) {
        const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(file) + w);
        if (!(((v & 0xFF) == 0xFF) | (((v >> 8) & 0xFF) == 0xFF) | (((v >> 16) & 0xFF) == 0xFF) | ((v >> 24) == 0xFF)))
            continue;
        for (int k = 0; k < 4; ++k) {
            const int64_t i = 4 * w + k;
            if (i < first || i + 1 >= nbytes || ((v >> (8 * k)) & 0xFF) != 0xFF || (file[i + 1] & 0xFE) != 0xF8) continue;
            sbflac::Header h;
            if (sbflac::parse_header(file + i, nbytes - i, channels, bits, rate, &h) != sbflac::kOk) continue;
            const unsigned long long slot = atomicAdd(count, 1ull);
            if ((int64_t)slot < cap) {
                Candidate c; c.offset = i; c.number = h.number; c.block_size = h.block_size;
                c.assignment = (int16_t)h.assignment; c.variable = (int16_t)h.variable;
                out[slot] = c;
            }
        }
    }
}

// Frames listed by a container: one thread per frame parses the header at its listed offset, bounded by the next one
__global__ void __launch_bounds__(256)
k_flac_frames(const uint8_t* __restrict__ buf, int64_t nbytes, const int64_t* __restrict__ offsets, int64_t n,
              int channels, int bits, int rate, sbflac::ListedFrame* __restrict__ out) {
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f < n) out[f] = sbflac::listed_frame(buf, nbytes, offsets, n, f, channels, bits, rate);
}

__global__ void __launch_bounds__(64)
k_flac_decode(const uint8_t* __restrict__ file, const FrameDesc* __restrict__ frames, int64_t n_frames, int channels,
              int bits, int rate, int32_t* __restrict__ planar, sbflac::FrameStatus* __restrict__ status) {
    __shared__ uint16_t s_crc[256];
    for (int i = threadIdx.x; i < 256; i += blockDim.x) s_crc[i] = sbflac::crc16_entry(i);
    __syncthreads();
    const int64_t f = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n_frames) return;
    const FrameDesc d = frames[f];
    sbflac::FrameStatus st;
    st.pad = 0;
    st.code = sbflac::decode_frame(file, d.offset, d.limit, channels, bits, rate, s_crc, planar + d.sample * channels,
                                   &st.end);
    status[f] = st;
}

__global__ void __launch_bounds__(256)
k_flac_decorrelate(const FrameDesc* __restrict__ frames, int64_t n_frames, int channels, int bits,
                   const int32_t* __restrict__ planar, int16_t* __restrict__ pcm) {
    for (int64_t f = blockIdx.x; f < n_frames; f += gridDim.x) {
        const FrameDesc d = frames[f];
        const int32_t* in = planar + d.sample * channels;
        for (int j = threadIdx.x; j < d.block_size; j += blockDim.x)
            sbflac::decorrelate(in, d.block_size, j, channels, d.assignment, bits, pcm + (d.sample + j) * channels);
    }
}

}  // namespace

namespace {

// A FLAC input on the device and its frame table while it is decoded; the upload is freed with it
struct FlacInput {
    Blocks blocks;
    const uint8_t* d_file = nullptr;
    int64_t nbytes = 0;
    int channels = 0, bits = 0, framerate = 0;
    std::vector<FrameDesc> frames;
    const int64_t* where = nullptr;    // sb_flac_decode_frames: file offset of each frame's block (messages name it)
    int64_t samples = 0;
};

// k_flac_decode, the frame checks, k_flac_decorrelate: the int16 PCM of every frame of h.frames
int decode(const FlacInput& h, sb_pcm** out, const char* who) {
    Ctx& c = ctx();
    const int64_t nf = (int64_t)h.frames.size();
    const int ch = h.channels;
    Blocks blocks;
    FrameDesc* d_frames = nullptr;
    int32_t* d_planar = nullptr;
    int16_t* d_pcm = nullptr;
    sbflac::FrameStatus* d_status = nullptr;
    SB_TRY(blocks.alloc(&d_frames, (size_t)nf));
    SB_TRY(blocks.alloc(&d_planar, (size_t)h.samples * ch));
    SB_TRY(blocks.alloc(&d_pcm, (size_t)h.samples * ch));
    SB_TRY(blocks.alloc(&d_status, (size_t)nf));
    std::vector<sbflac::FrameStatus> status((size_t)nf);
    cudaError_t e = cudaMemcpyAsync(d_frames, h.frames.data(), sizeof(FrameDesc) * nf, cudaMemcpyHostToDevice, c.stream);
    if (e == cudaSuccess && nf > 0) {
        ProfScope ps("flac_decode");
        k_flac_decode<<<(unsigned)((nf + 63) / 64), 64, 0, c.stream>>>(h.d_file, d_frames, nf, ch, h.bits, h.framerate,
                                                                       d_planar, d_status);
        e = cudaGetLastError();
    }
    SB_TRY(collect(e, status.data(), d_status, nf, who));
    // every frame must decode, pass its CRC-16 and end exactly where the next frame (or the file) does
    char msg[256];
    auto bytes_at = [&](int64_t off, uint8_t* buf) {
        if (off < h.nbytes) cudaMemcpy(buf, h.d_file + off, (size_t)std::min<int64_t>(16, h.nbytes - off), cudaMemcpyDeviceToHost);
    };
    if (!sbflac::check_frames(h.frames, status.data(), h.nbytes, ch, h.bits, h.framerate, bytes_at, msg, sizeof(msg),
                              h.where))
        SB_FAIL(SB_EINVAL, "%s", msg);
    if (nf > 0) {
        ProfScope ps("flac_decorrelate");
        k_flac_decorrelate<<<(unsigned)std::max<int64_t>(1, std::min<int64_t>(nf, (int64_t)c.sm_count * 64)), 256, 0,
                             c.stream>>>(d_frames, nf, ch, h.bits, d_planar, d_pcm);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c.stream);
    SB_TRY(cuda_result(e, who));
    return pcm_handle(blocks.take(d_pcm), h.samples, ch, h.framerate, out);
}

// the stream parameters, and the listed frames: a frame ends where the next one starts, so the frame named is the one
// that starts at or before its predecessor
int check_listed(const int64_t* offsets, const int64_t* file_offsets, int64_t n, int64_t nbytes, int channels, int bits,
                 int framerate, const char* who) {
    if (bits != 16 && bits != 24) SB_FAIL(SB_EINVAL, "FLAC with %d bits per sample is not supported (16 or 24)", bits);
    if (channels < 1 || channels > 8 || framerate < 1 || nbytes < 1 || n < 0)
        SB_FAIL(SB_EINVAL, "%s: bad stream parameters", who);
    for (int64_t f = 0; f < n; ++f)
        if (offsets[f] < 0 || offsets[f] >= nbytes || (f > 0 && offsets[f] <= offsets[f - 1]))
            SB_FAIL(SB_EINVAL, "FLAC frame %lld at byte offset %lld: %s", (long long)f, (long long)file_offsets[f],
                    offsets[f] < 0 || offsets[f] >= nbytes ? "frame starts outside the buffer" : "empty frame");
    return SB_OK;
}

// after check_listed: k_flac_frames on the listed frames, their table, then decode
int decode_listed(const uint8_t* d_buf, int64_t nbytes, const int64_t* d_offsets, const int64_t* offsets,
                  const int64_t* file_offsets, int64_t n, int channels, int bits, int framerate, sb_pcm** out,
                  const char* who) {
    Ctx& c = ctx();
    FlacInput h;
    h.d_file = d_buf;
    h.nbytes = nbytes; h.channels = channels; h.bits = bits; h.framerate = framerate;
    h.where = file_offsets;
    std::vector<sbflac::ListedFrame> listed((size_t)n);
    {
        Blocks blocks;
        sbflac::ListedFrame* d_listed = nullptr;
        SB_TRY(blocks.alloc(&d_listed, (size_t)n));
        cudaError_t e = cudaSuccess;
        if (n > 0) {
            ProfScope ps("flac_frames");
            k_flac_frames<<<(unsigned)((n + 255) / 256), 256, 0, c.stream>>>(d_buf, nbytes, d_offsets, n, channels,
                                                                             bits, framerate, d_listed);
            e = cudaGetLastError();
        }
        SB_TRY(collect(e, listed.data(), d_listed, n, who));
    }
    char msg[256];
    if (!sbflac::list_frames(listed.data(), offsets, file_offsets, n, nbytes, h.frames, &h.samples, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return decode(h, out, who);
}

}  // namespace

namespace sb {

int flac_decode(const uint8_t* d_buf, int64_t nbytes, const int64_t* d_offsets, const int64_t* offsets,
                const int64_t* file_offsets, int64_t n, int channels, int bits, int framerate, sb_pcm** out,
                const char* who) {
    SB_TRY(check_listed(offsets, file_offsets, n, nbytes, channels, bits, framerate, who));
    return decode_listed(d_buf, nbytes, d_offsets, offsets, file_offsets, n, channels, bits, framerate, out, who);
}

}  // namespace sb

extern "C" {

int sb_flac_decode_file(const void* file, int64_t nbytes, int64_t first_frame_offset, int channels, int bits,
                        int framerate, sb_pcm** out) {
    const char* who = "sb_flac_decode_file";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, file && out));
    if (bits != 16 && bits != 24) SB_FAIL(SB_EINVAL, "FLAC with %d bits per sample is not supported (16 or 24)", bits);
    if (channels < 1 || channels > 8 || framerate < 1 || nbytes < 1 || first_frame_offset < 0 || first_frame_offset > nbytes)
        SB_FAIL(SB_EINVAL, "sb_flac_decode_file: bad stream parameters");
    FlacInput h;
    h.nbytes = nbytes; h.channels = channels; h.bits = bits; h.framerate = framerate;
    const uint8_t* host = static_cast<const uint8_t*>(file);
    uint8_t* d_file = nullptr;
    SB_TRY(upload_padded(h.blocks, &d_file, file, nbytes, who));
    h.d_file = d_file;

    // candidates: a frame has at least 9 bytes; real files hold one frame per few kB and false syncs are rarer still
    std::vector<Candidate> cand;
    SB_TRY(scan_candidates(nbytes / 256 + 4096, "flac_sync", who, [&](Candidate* d_cand, unsigned long long* d_count, int64_t cap) {
        const int64_t words = (nbytes + 3) / 4;
        const int grid = (int)std::min<int64_t>((words + 255) / 256, (int64_t)c.sm_count * 16);
        k_flac_sync<<<std::max(grid, 1), 256, 0, c.stream>>>(h.d_file, first_frame_offset, nbytes, channels, bits,
                                                             framerate, d_cand, d_count, cap);
    }, cand));
    char msg[256];
    if (!sbflac::chain(cand, first_frame_offset, nbytes, channels, bits, framerate, host + first_frame_offset, h.frames,
                       &h.samples, msg, sizeof(msg)))
        SB_FAIL(SB_EINVAL, "%s", msg);
    return decode(h, out, who);
}

int sb_flac_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                          int channels, int bits, int framerate, sb_pcm** out) {
    const char* who = "sb_flac_decode_frames";
    Ctx& c = ctx();
    SB_TRY(entry_check(who, buf && offsets && file_offsets && out));
    SB_TRY(check_listed(offsets, file_offsets, n, nbytes, channels, bits, framerate, who));
    Blocks blocks;
    uint8_t* d_buf = nullptr;
    int64_t* d_offsets = nullptr;
    SB_TRY(upload_padded(blocks, &d_buf, buf, nbytes, who));
    SB_TRY(blocks.alloc(&d_offsets, (size_t)n));
    SB_TRY(cuda_result(cudaMemcpyAsync(d_offsets, offsets, sizeof(int64_t) * n, cudaMemcpyHostToDevice, c.stream), who));
    return decode_listed(d_buf, nbytes, d_offsets, offsets, file_offsets, n, channels, bits, framerate, out, who);
}

}  // extern "C"
