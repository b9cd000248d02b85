/*
 * sushi_b200.h -- C ABI of the H100-native audio template-matching library.
 *
 * This is the drop-in boundary for ONE path of tp7/Sushi: the per-event audio
 * template match that the reference performs in Python through OpenCV,
 *
 *     WavStream.get_substream / find_substream      reference wav.py:168-188
 *     cv2.matchTemplate(..., TM_SQDIFF_NORMED)      reference wav.py:185
 *     result.argmin(axis=1)[0]                      reference wav.py:186
 *     load-time downsample / pad / normalise        reference wav.py:64-91,108-156
 *
 * The reference has no FFI of its own (it is pure Python calling cv2), so these
 * entry points are what a ctypes binding inside the reference's wav.py would
 * call (see INTEGRATION.md for that stub).  Conventions:
 *
 *   - plain C: pointers, sizes, integer sample offsets.  All time -> sample
 *     conversion (wav.py:173-175) stays on the Python side so that it is
 *     reproduced bit-for-bit; the C side never sees seconds.
 *   - every call returns SB_OK (0) or a negative SB_E* code; the text of the
 *     last failure on the calling thread is available from sb_last_error().
 *   - the caller owns every host buffer; the library owns device memory behind
 *     opaque handles.  One host thread drives one GPU (one process per GPU).
 *   - blocking calls return after their results are in the caller's host
 *     buffers.  *_device variants take/return device pointers and only enqueue
 *     work on the library stream (sb_sync() waits for it).
 *
 * Result convention (mirrors wav.py:185-188): for a query with template length
 * n and nlags candidate positions, curve[j] is OpenCV's TM_SQDIFF_NORMED value
 * of the template against image[lag0+j .. lag0+j+n), j in [0, nlags), rounded
 * to float32; the call returns diff = min_j curve[j] and idx = the FIRST j that
 * attains it (numpy argmin rule).
 */
#ifndef SUSHI_B200_H
#define SUSHI_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_ABI_VERSION 18

/* status codes */
#define SB_OK            0
#define SB_EINVAL       -1   /* bad argument (range, NULL, dtype)            */
#define SB_ECUDA        -2   /* CUDA runtime failure                         */
#define SB_ENOMEM       -3   /* host or device allocation failed             */
#define SB_ESTATE       -4   /* library not initialised / already shut down  */

/* sample types of a resident stream (reference wav.py:108-110,153-156) */
#define SB_U8  0             /* 'uint8'   : reference default (sushi.py:769) */
#define SB_F32 1             /* 'float32'                                    */

typedef struct sb_stream sb_stream;      /* opaque: one normalised stream in HBM */
typedef struct sb_pcm sb_pcm;            /* opaque: decoded interleaved int16 PCM on the device */
typedef struct sb_ts sb_ts;              /* opaque: one audio PID of an MPEG transport stream being demuxed */
typedef struct sb_ps sb_ps;              /* opaque: one audio stream of an MPEG program stream being demuxed */
typedef struct sb_ogg sb_ogg;            /* opaque: one FLAC stream of an Ogg file being demuxed */
typedef struct sb_avi sb_avi;            /* opaque: one audio stream of an AVI file being demuxed */

/* ---- life cycle ------------------------------------------------------- */

/* Bind the calling process to CUDA device `device` and create the library
 * stream and scratch.  Idempotent for the same device. */
int sb_init(int device);
int sb_shutdown(void);
/* ABI version of the loaded library (compare with SB_ABI_VERSION). */
int sb_abi_version(void);
/* Text of the last error on this thread ("" if none). Never NULL. */
const char* sb_last_error(void);
/* Wait until everything enqueued on the library stream has finished. */
int sb_sync(void);
/* Lag-block size in samples.  Every engine runs at 16384 (the FFT size is twice that); sb_set_block_size
 * accepts 16384 and fails with SB_EINVAL for anything else. */
int sb_set_block_size(int block);
int sb_get_block_size(void);
/* Engine behind sb_find*:
 *   2 (default) = the packed fused lag-block kernels (sb_fused2.cu): spectral multiply, inverse FFT in
 *       shared memory, normalisation and argmin in one launch, on spectra stored in a paired layout;
 *       templates of 12+ partitions keep engine 1's blocked multiply.  One CTA handles one lag block, or
 *       (batches averaging >= 4 template partitions) a pair of consecutive lag blocks that share their
 *       template rows, the second product spectrum waiting in an L2-resident scratch; both give
 *       bit-identical results;
 *   4 / 5 = engine 2 with pairs always / never;
 *   1 = the first fused lag-block kernel (sb_fused.cu).
 * Any other value fails with SB_EINVAL.  Engines agree to float32 FFT rounding (~2e-7 of the curve), not
 * bit for bit. */
int sb_set_engine(int engine);
int sb_get_engine(void);
/* Spectral multiply, every engine: 0 (default) = per lag block inside the fused kernel, except for
 * queries whose template spans 12 or more partitions (>= 16.4 s at 12 kHz), which go through the
 * register-blocked multiply kernel (8 lag blocks share each template row) and engine 1's fused kernel;
 * 1 = never blocked, 2 = always blocked.  The route depends only on the query, not on the rest of the
 * batch. */
int sb_set_premac_mode(int mode);
/* Overlap-save geometry: every engine runs at hop B (template partitions of B samples, half of each
 * inverse FFT is valid lags).  sb_set_hop_mode accepts 1 (hop B) and fails with SB_EINVAL for anything
 * else. */
int sb_set_hop_mode(int mode);
/* Body variant of the packed kernels (engines 2, 4, 5) on uint8 streams: 3 (default) = per run of 8 lags a lower
 * and an upper bound of the screening values from the run's largest correlation value and its exact head sums; only
 * the runs whose lower bound does not exceed the lag block's smallest upper bound can hold the minimum -- they leave
 * the match kernel as records (query, first lag, 8 correlation values) and a second kernel evaluates their lags in
 * fp64; window sums slide on the staged sample windows, per-query constants travel through shared memory, the
 * self-mirrored quad is prefetched; 1 = the first version (fp32 screening of every lag and fp64 evaluation of the
 * candidates inside the match kernel, running sums read from HBM).  Either way the result is the fp64 evaluation of
 * every lag that can be the minimum, so the two agree bit for bit (checked on the GPU by the test-suite); float32
 * streams and the other engines ignore the setting.  (2, the per-lag loop of 3 run over all lags, was measured and
 * dropped in round 2.) */
int sb_set_epilogue(int variant);
int sb_get_epilogue(void);
/* Template partition spectra kept resident per pass over a batch (>= 1); batches needing more are
 * processed in several passes of whole queries. */
int sb_set_max_parts(int64_t parts);

/* The library's CUDA stream (a cudaStream_t) so that a host framework can order its own
 * work (e.g. an NCCL broadcast issued through torch.distributed) on the same stream. */
void* sb_get_stream(void);
/* Page-locked host buffers for callers that want true asynchronous H2D/D2H copies. */
int sb_pinned_alloc(int64_t bytes, void** out);
int sb_pinned_free(void* p);

/* Plain device buffers for callers that keep results on the GPU (sb_find_batch_device). */
int sb_device_alloc(int64_t bytes, void** out);
int sb_device_free(void* p);
int sb_copy_to_host(void* host_dst, const void* dev_src, int64_t bytes);   /* ordered on the library stream, blocking */
int sb_copy_to_device(void* dev_dst, const void* host_src, int64_t bytes); /* ordered on the library stream, blocking */
int sb_copy_on_device(void* dev_dst, const void* dev_src, int64_t bytes);  /* enqueued on the library stream */

/* ---- resident streams:  WavStream.data  (wav.py:119,140-156) ----------- */

/* Upload a normalised stream of n samples (dtype SB_U8 or SB_F32) from host
 * memory, build its running sums (the integral image cv2 builds per call,
 * wav.py:185) and keep it resident.  */
int sb_stream_create(const void* host_samples, int64_t n, int dtype, sb_stream** out);
/* Same, but `dev_samples` is already a device pointer on the bound GPU (e.g.
 * the receive buffer of an NCCL broadcast); it is copied device-to-device. */
int sb_stream_create_device(const void* dev_samples, int64_t n, int dtype, sb_stream** out);
int sb_stream_destroy(sb_stream* s);
/* Device address of the raw samples of a resident stream (read-only for the caller). */
const void* sb_stream_device_ptr(const sb_stream* s);
int64_t sb_stream_length(const sb_stream* s);
int sb_stream_dtype(const sb_stream* s);
/* Copy samples [off, off+n) back to host (tests, WavStream.data mirror). */
int sb_stream_read(const sb_stream* s, int64_t off, int64_t n, void* host_out);

/* ---- the matcher:  WavStream.find_substream  (wav.py:177-188) ---------- */

/* One query whose template is a raw host array (pattern is "any (1,n)
 * ndarray", e.g. np.split halves, sushi.py:445).  dtype must equal the image
 * stream's.  Template bytes are uploaded inside the call. */
int sb_find(const sb_stream* image, const void* tmpl_host, int64_t tmpl_len,
            int64_t lag0, int64_t nlags, float* diff_out, int64_t* idx_out);

/* `count` independent queries; template q = tmpl[tmpl_off[q] .. +tmpl_len[q])
 * (get_substream as an (offset,length) descriptor: no bytes move,
 * wav.py:168-171), searched over image positions [lag0[q], lag0[q]+nlags[q]).
 * Requirements per query: tmpl_len>=1, nlags>=1,
 * tmpl_off+tmpl_len <= len(tmpl), lag0>=0, lag0+nlags-1+tmpl_len <= len(image).
 * image and tmpl may be the same stream.  Host arrays in, host arrays out. */
int sb_find_batch(const sb_stream* image, const sb_stream* tmpl, int64_t count,
                  const int64_t* tmpl_off, const int64_t* tmpl_len,
                  const int64_t* lag0, const int64_t* nlags,
                  float* diff_out, int64_t* idx_out);

/* Same queries (descriptor arrays still in HOST memory: they are planned on the
 * host), but the two result arrays are DEVICE pointers and the call only
 * enqueues work on the library stream (no host synchronisation; sb_sync()
 * waits).  Used by the multi-GPU path, where the per-rank results feed an NCCL
 * all-gather without a round trip through the host. */
int sb_find_batch_device(const sb_stream* image, const sb_stream* tmpl, int64_t count,
                         const int64_t* tmpl_off, const int64_t* tmpl_len,
                         const int64_t* lag0, const int64_t* nlags,
                         float* d_diff_out, int64_t* d_idx_out);

/* Whole curves of `count` queries, concatenated in query order into curves_out[sum(nlags)] (host).
 * Every lag is evaluated with the exact fp64 rule.  Because a value depends only on (template,
 * absolute position), a curve over a wider range answers any sub-range query exactly: the shift
 * solver uses this to precompute the next groups' searches in one launch (sushi_b200/shifts.py). */
int sb_match_curves(const sb_stream* image, const sb_stream* tmpl, int64_t count,
                    const int64_t* tmpl_off, const int64_t* tmpl_len,
                    const int64_t* lag0, const int64_t* nlags, float* curves_out);
/* ---- many streams in one call (ABI version 2) ------------------------------
 *
 * The same queries as sb_find_batch / sb_match_curves, but every query names its own image and template stream:
 * query q matches streams[tmpl_slot[q]][tmpl_off[q] .. +tmpl_len[q]) against streams[image_slot[q]] over positions
 * [lag0[q], lag0[q]+nlags[q]).  A value depends only on (template, absolute position), so queries of different
 * streams -- different episodes of a season -- share one launch without changing any result: each result equals what
 * sb_find_batch / sb_match_curves return for that query alone, bit for bit.  Per-query rules are theirs, checked
 * against the query's own streams.  All streams must share one sample type and carry running sums; a NULL entry,
 * a slot outside [0, n_streams), a stream without running sums or mixed sample types fail with SB_EINVAL, and
 * sb_last_error() names the query or slot.
 * The packed engine (2, 4, 5) runs the whole call in one set of launches whatever the number of streams; queries of
 * the blocked class (templates of 12+ partitions) and engine 1 run as one sb_find_batch-like pass per distinct
 * (image, template) pair inside the call. */
int sb_find_multi(const sb_stream* const* streams, int32_t n_streams, int64_t count,
                  const int32_t* image_slot, const int32_t* tmpl_slot,
                  const int64_t* tmpl_off, const int64_t* tmpl_len,
                  const int64_t* lag0, const int64_t* nlags,
                  float* diff_out, int64_t* idx_out);
/* Whole curves of the queries above, concatenated in query order into curves_out[sum(nlags)] (host). */
int sb_match_curves_multi(const sb_stream* const* streams, int32_t n_streams, int64_t count,
                          const int32_t* image_slot, const int32_t* tmpl_slot,
                          const int64_t* tmpl_off, const int64_t* tmpl_len,
                          const int64_t* lag0, const int64_t* nlags, float* curves_out);

/* The whole curve of one query (debug / parity tests): curve_out[nlags]. */
int sb_match_curve(const sb_stream* image, const sb_stream* tmpl,
                   int64_t tmpl_off, int64_t tmpl_len, int64_t lag0, int64_t nlags,
                   float* curve_out);

/* ---- the loader:  WavStream.__init__  (wav.py:64-91,108-156) ----------- */

/* Decode interleaved PCM (sample_width 2 = int16 LE, 3 = int24 LE top 16 bits,
 * wav.py:68-74), average `channels` channels (wav.py:80-90) and resample each
 * READ_CHUNK (= `framerate` frames) with OpenCV's INTER_NEAREST index map
 * (wav.py:125-137) into a padded float32 buffer of total_len samples whose
 * first `padding` samples and last `padding` samples repeat the edge values
 * (wav.py:140-141).  Output stays on the device behind `*out_f32` (a SB_F32
 * stream holding the UN-normalised samples). */
int sb_load_pcm(const void* pcm_host, int64_t frames, int channels, int sample_width,
                int framerate, int sample_rate, int64_t padding, int64_t total_len,
                sb_stream** out_f32);
/* Median-clip normalise (wav.py:145-151) and optionally quantise to uint8
 * (wav.py:153-156) a stream produced by sb_load_pcm; returns a new resident
 * stream of dtype `dtype` ready for sb_find*.  min3/max3 (3 x the medians) are
 * returned for the host mirror. */
int sb_normalise(const sb_stream* raw_f32, int dtype, sb_stream** out,
                 float* min3_out, float* max3_out);

/* ---- decoded input (ABI version 9) -------------------------------------------
 *
 * Every compressed input loads exactly as the plain PCM WAV of its decoded samples loads through sb_load_pcm.  A
 * decoder is one call: it uploads the input, decodes it on the GPU, checks it completely and returns an sb_pcm
 * handle, the decoded interleaved int16 PCM on the device (24-bit and wider samples keep their top 16 bits).  A
 * damaged input fails with SB_EINVAL, sb_last_error() naming the frame or access unit and its byte offset, and no
 * handle is returned.  The stream geometry stays with the caller, as it does for WAV: sb_pcm_info gives the sample
 * frames, channels and rate it needs, and sb_pcm_load resamples to sample_rate and pads exactly as sb_load_pcm does,
 * into a SB_F32 stream for sb_normalise.  The handle may be loaded any number of times until sb_pcm_destroy. */
int sb_pcm_info(const sb_pcm* pcm, int64_t* frames, int32_t* channels, int32_t* rate);
int sb_pcm_load(const sb_pcm* pcm, int sample_rate, int64_t padding, int64_t total_len, sb_stream** out_f32);
int sb_pcm_destroy(sb_pcm* pcm);

/* Big-endian 16- or 24-bit interleaved PCM (QuickTime `twos` / `in24`, ISO `ipcm`): loaded through sb_pcm_load it
 * gives bit for bit what sb_load_pcm gives on the byte-swapped data. */
int sb_pcm_from_be(const void* pcm_host, int64_t frames, int channels, int sample_width, int framerate, sb_pcm** out);

/* Little-endian 16- or 24-bit interleaved PCM (ABI version 12; Matroska `A_PCM/INT/LIT`, MP4 `sowt` / `lpcm`): the
 * top 16 bits of each sample, as sb_load_pcm reads them. */
int sb_pcm_from_le(const void* pcm_host, int64_t frames, int channels, int sample_width, int framerate, sb_pcm** out);

/* The ffmpeg command line's `-ac 1 -ar <out_rate> -acodec pcm_s16le` on S16 audio (ABI version 12): a new mono
 * handle at out_rate holding what libswresample 6.1.100 with its default options gives on its x86-64 FMA3 path, bit
 * for bit and frame for frame.  `layout` is FFmpeg's channel mask of the input (AV_CH_*; its bit count is the
 * handle's channel count).  Equal rates take the integer Q15 downmix and a mono input is copied; otherwise every
 * channel is resampled in float by the Kaiser-windowed polyphase filter and then remixed.  Fails on a layout
 * libswresample refuses or with channels other than FL FR FC LFE BL BR FLC FRC BC SL SR, and on a rate pair whose
 * filter window exceeds 48 KB of shared memory per 32 outputs.  `in` is left as it is. */
int sb_pcm_swr(const sb_pcm* in, uint64_t layout, int out_rate, sb_pcm** out);

/* FLAC (ABI version 3).  16 and 24 bits per sample and 1 to 8 channels are accepted; the caller has read STREAMINFO
 * and passes its channel count, bits per sample and sample rate.  Every frame must decode, pass its CRC-16 and end
 * exactly where the next frame (or the input) does.  The STREAMINFO MD5 is not checked.
 * sb_flac_decode_file takes the whole file (`nbytes` bytes, metadata included) and finds its frames: the first at
 * first_frame_offset, each next one by its coded frame or sample number.
 * sb_flac_decode_frames (ABI version 5) takes frames a container lists.  `buf` holds a track's frame payloads back to
 * back (`nbytes` bytes, no metadata); frame f starts at offsets[f] (increasing) and ends exactly where frame f + 1
 * starts, the last at nbytes.  file_offsets[f] is the byte offset in the container file of the block holding frame
 * f: every error names it.  Each header must parse, agree with the stream parameters and pass its CRC-8 at its listed
 * offset.  The coded frame / sample numbers are not checked (a cut track starts above 0), and sample positions follow
 * from the block sizes. */
int sb_flac_decode_file(const void* file, int64_t nbytes, int64_t first_frame_offset, int channels, int bits,
                        int framerate, sb_pcm** out);
int sb_flac_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                          int channels, int bits, int framerate, sb_pcm** out);

/* Dolby TrueHD (ABI version 6): FFmpeg's decoder output, channels in FFmpeg's order, the presentation of substream
 * min(n - 1, 2) (a fourth, object substream is skipped).  `buf` holds the stream's bytes (`nbytes`); a container's
 * blocks start at offsets[0..n) (increasing, back to back; a raw .thd stream is one block at 0) and file_offsets[b]
 * is the byte offset in the file of block b, which errors name (a negative one: errors name the AU's own offset, as
 * for a raw stream).  An access unit (AU) must end inside its block.  The call lists the major syncs on the GPU,
 * chains the AUs into restart segments on the host and decodes every segment on the GPU, one thread each.  It fails on
 * any damage listed in DESIGN.md section 2: check nibble, major sync CRC, restart header checksum, substream parity or
 * CRC, lossless check, AU lengths, a segment without restart headers, a short AU before the end.  MLP is refused. */
int sb_truehd_decode(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                     sb_pcm** out);

/* ALAC, Apple Lossless (ABI version 8): FFmpeg's `alac` decoder output, 20-, 24- and 32-bit samples by the top 16
 * bits of FFmpeg's S32 sample, channels in FFmpeg's order.  `buf` holds the track's frames back to back (`nbytes`
 * bytes): frame f starts at offsets[f] (increasing) and ends where frame f + 1 starts, the last at nbytes.
 * file_offsets[f] is the byte offset in the container file of the MP4 sample or Matroska block holding frame f: every
 * error names it with the frame index.  config[0..6] is the ALACSpecificConfig: frameLength (1 to 65536), bitDepth
 * (16, 20, 24, 32), pb, mb, kb, channels (1 to 8), sampleRate.  One GPU thread decodes each frame.  It fails on: an
 * element tag other than SCE, CPE, LFE and END; more or fewer channels than the config declares; a sample count of 0
 * or above frameLength, or differing between elements; a prediction type other than 0 and 15; an invalid element
 * header; a frame that reads past its bytes; a frame without END.  Bytes after END are ignored. */
int sb_alac_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                          const int32_t* config, sb_pcm** out);

/* WavPack (ABI version 10): FFmpeg's `wavpack` decoder output for lossless integer streams of 2 or 3 bytes per sample,
 * 3-byte samples by the top 16 bits of FFmpeg's S32 sample, channels in FFmpeg's order (blocks in order within a
 * frame).  `buf` holds the stream's blocks (`nbytes` bytes); table holds 8 int64 per block b: the offset and size of
 * its metadata sub-blocks in buf, block_samples (1 to 150000), the header's flags and CRC, the track sample where the
 * block starts, its first output channel (a block fills one channel when its flags say mono, two otherwise), and the
 * byte offset in the file of the block's header (.wv) or Matroska block, which every error names with the block index.
 * The host builds the table from the block headers and checks their sequence; `channels` (1 to 8) and `rate` are the
 * stream's.  One GPU thread decodes each block.  It fails on: hybrid, float, DSD or 1- / 4-byte flags; a sub-block
 * that runs past its block; samples without ID_WV_BITSTREAM, or without terms, weights, sample history or medians;
 * more than 16 decorrelation terms or an invalid one; invalid weights, sample history, medians, ID_INT32_INFO or
 * ID_SAMPLE_RATE; extended precision (ID_WVX_BITSTREAM, ID_INT32_INFO sent bits); a mono block without terms; a
 * bitstream that reads past its sub-block; a 16-bit stereo sample above 2^19; a block CRC that disagrees. */
int sb_wavpack_decode_blocks(const void* buf, int64_t nbytes, const int64_t* table, int64_t n, int32_t channels,
                             int32_t rate, sb_pcm** out);

/* TTA, True Audio (ABI version 11): FFmpeg's `tta` decoder output for format-1 streams of 16 or 24 bits, 24-bit
 * samples by the top 16 bits of FFmpeg's S32 sample, channels in FFmpeg's order.  `buf` holds the stream's frames back
 * to back (`nbytes` bytes): frame f starts at offsets[f] (increasing) and ends where frame f + 1 starts, the last at
 * nbytes; each ends with the CRC-32 of its bitstream.  file_offsets[f] is the byte offset in the file of the frame
 * (.tta) or of the Matroska block holding it: every error names it with the frame index.  config[0..4] is channels (1
 * to 8), bits (16 or 24), rate (1 to 2^23 - 1), the frame length (256 * rate / 245) and the last frame's length (0 when
 * it is a whole frame); every other frame holds a whole frame.  One GPU thread decodes each frame.  It fails on: a
 * unary run or a code that reads past the frame's bitstream; a Rice parameter above 25; a frame other than the last
 * that reaches the last frame's length with only its CRC left (FFmpeg's decoder cuts such a frame short); bytes left
 * between the last sample and the CRC; a CRC that disagrees. */
int sb_tta_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                         const int32_t* config, sb_pcm** out);

/* Monkey's Audio, APE (ABI version 16): FFmpeg's `ape` decoder output for file version 3990 (Monkey's Audio 3.99 and
 * later), compression levels 1000 to 5000, 16 or 24 bits, mono or stereo; 24-bit samples by the top 16 bits of
 * FFmpeg's S32 sample.  `buf` holds the file's bytes up to `nbytes` (the file less its stored WAV tail): frame f starts
 * at offsets[f] (its seek-table position plus any ID3v2 tag in front; increasing), and, as FFmpeg's demuxer cuts it,
 * runs to the next frame's start, the last to nbytes; the frames are 32-bit little-endian words counted from frame 0.
 * file_offsets[f] is what an error names with the frame index.  config[0..5] is channels (1 or 2), bits (16 or 24),
 * rate, compression level, blocks per frame and the last frame's blocks.  The decode runs in stages over an int32
 * scratch of every sample: the range decoder (one thread per frame), the NN filters (one warp per frame and channel),
 * the predictor (one thread per frame) and the frame CRC (one warp per frame).  It fails on: a frame header cut short;
 * frame flags other than mono silence, stereo silence and pseudo-stereo; a range decoder that reads past its frame or
 * meets a symbol past 65535; a CRC that disagrees (FFmpeg checks it only under AV_EF_CRCCHECK); a 24-bit stereo sample
 * past 24 bits (where FFmpeg switches to its 64-bit predictor). */
int sb_ape_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets, int64_t n,
                         const int32_t* config, sb_pcm** out);

/* TAK (ABI version 17): FFmpeg's `tak` decoder output for integer TAK of 16 or 24 bits, 1 to 6 channels, codec types
 * mono/stereo and multichannel; 24-bit samples by the top 16 bits of FFmpeg's S32 sample.  `file` holds the whole
 * file (nbytes bytes); its frames lie in [audio_start, audio_end) (audio_end: LAST_FRAME's end, a trailing APEv2 or
 * ID3v1 tag, or the end of the file).  config[0..7] is channels, bits, rate, codec type, frame size type, the total
 * samples per channel (low and high 32 bits) and the channel mask, all from STREAMINFO.  Frames start where FFmpeg's
 * tak parser starts them (sync word, a header that parses, its CRC-24), found on the GPU; they must be numbered from
 * 0, start at audio_start and follow each other with no byte between, the first carry stream info, every stream info
 * agree with config, and the lengths add up to the total.  The decode runs in stages over an int32 scratch of every
 * sample: the residual codes (one thread per frame), the prediction filters (one warp per frame and channel), the
 * decorrelation, lpc scans and store (one CTA per frame) and the data CRC (one warp per frame).  It fails, naming the
 * frame and its byte offset, on: a read past the frame; a subframe layout, filter order or residual coding FFmpeg
 * rejects; a sample shift at or above the bit depth; filtered decorrelation on fewer than 256 samples; multichannel
 * decorrelation parameters FFmpeg rejects or that leave a channel undecoded; the frame metadata flag; bytes after the
 * data CRC; a data CRC that disagrees (FFmpeg checks it only under AV_EF_CRCCHECK). */
int sb_tak_decode_file(const void* file, int64_t nbytes, int64_t audio_start, int64_t audio_end, const int32_t* config,
                       sb_pcm** out);

/* MPEG-1/2 audio layer II, MP2 (ABI version 13): FFmpeg's fixed-point `mp2` decoder output, bit for bit, 1 or 2
 * channels at 16 to 48 kHz.  `buf` holds a Matroska track's block payloads back to back (block k at offsets[k], at
 * file offset file_offsets[k]).  FFmpeg decodes each block as a packet, so every block must start with a frame header
 * and hold whole frames; a last frame cut short is decoded with zeros for its missing bits, as FFmpeg decodes it.
 * Refused with SB_EINVAL, naming the frame and the file offset of its block: layer I or III, MPEG-2.5, free format, a
 * reserved bitrate, rate or emphasis, a broken sync, a change of layer, rate or channel count (bitrates may change), a
 * CRC-16 that disagrees, a frame whose samples run past its end, a frame that straddles blocks. */
int sb_mp2_decode_frames(const void* buf, int64_t nbytes, const int64_t* offsets, const int64_t* file_offsets,
                         int64_t n, sb_pcm** out);
/* One MPEG audio stream as a raw .mp2 file holds it (ABI version 14): `buf` the bytes between the file's tags, which
 * start at file offset `file_offset`.  Split at its headers as FFmpeg's parser splits it, with SB_TS_MP2's rules: bytes
 * before the first header take the first whole frame with them (FFmpeg's decoder refuses that packet), and a last frame
 * cut short is decoded with zeros and sets *cut.  Refusals as sb_mp2_decode_frames's, naming the frame's own file
 * offset. */
int sb_mp2_decode_stream(const void* buf, int64_t nbytes, int64_t file_offset, int32_t* cut, sb_pcm** out);

/* ---- MPEG transport streams (ABI version 7) ----------------------------------
 *
 * One audio PID of a BDAV (192-byte packets: a 4-byte arrival time stamp, then the 188-byte packet) or plain
 * (188-byte) transport stream, demuxed and decoded on the GPU.  The file is fed in chunks of whole packets, in order;
 * the host does no per-packet work.  For each chunk k_ts_scan checks every packet's sync byte and, for the PID's
 * packets, the transport error indicator, scrambling control, adaptation field length and continuity counter
 * (carried across chunks; discontinuity_indicator honoured); the PID's payload bytes and packet table are appended on
 * the device (the rest of the chunk is not kept).  sb_ts_finish parses every PES header (k_pes_index), checks
 * PES_packet_length against the bytes the PID carried and returns the decoded PCM as an sb_pcm:
 *   SB_TS_PCM_BLURAY  every PES's BD-LPCM header must give the first one's channel assignment, rate and bits; each
 *                     PES gives its whole sample frames (leftover bytes are ignored) and k_bdlpcm_decode writes int16
 *                     PCM (16-bit samples as they are, 24-bit samples their top 16 bits, the padding channel of an
 *                     odd channel count dropped), as FFmpeg's pcm_bluray decoder returns them; 20-bit samples are
 *                     refused, as FFmpeg's decoder refuses them;
 *   SB_TS_TRUEHD      the payloads of the PES packets FFmpeg routes to the TrueHD stream (every stream_id_extension
 *                     but 0x76, the AC-3 sub-stream) are one raw TrueHD stream, decoded as sb_truehd_decode decodes a
 *                     .thd file; AUs may straddle PES and TS packets;
 *   SB_TS_MP2         (ABI version 13) the PES payloads are one MPEG audio stream, decoded as sb_mp2_decode_frames
 *                     decodes a track's blocks, but as one stream split at its headers, as FFmpeg's parser splits it:
 *                     bytes before the first header take the first whole frame with them (FFmpeg's decoder refuses
 *                     that packet), and a last frame cut short is decoded with zeros and sets *cut.
 * Damage fails with SB_EINVAL, sb_last_error() naming the byte offset of the packet (TS damage), of the PES's first
 * packet (PES damage) or of the packet holding an AU's first byte (TrueHD damage).  A last PES shorter than its
 * PES_packet_length (a cut file) keeps its whole sample frames and sets *cut; one cut inside its header is dropped.
 * sb_ts_feed returns once the chunk is copied, so the caller may refill its buffer while the GPU scans it.  The sb_pcm
 * outlives the sb_ts. */
#define SB_TS_PCM_BLURAY 0
#define SB_TS_TRUEHD 1
#define SB_TS_MP2 2
int sb_ts_open(int packet_size, int32_t pid, int32_t codec, sb_ts** out);
int sb_ts_feed(sb_ts* ts, const void* host_chunk, int64_t nbytes, int64_t file_offset);
int sb_ts_finish(sb_ts* ts, int32_t* cut, sb_pcm** out);
int sb_ts_destroy(sb_ts* ts);

/* ---- MPEG program streams (ABI version 14) ------------------------------------
 *
 * One MPEG audio stream (stream id 0xC0 to 0xDF; substream_id -1) of an MPEG-1 or MPEG-2 program stream (VCD and SVCD
 * .mpg, DVD .vob, DVB recordings), demuxed on the GPU and decoded as SB_TS_MP2 decodes a PID.  The file is fed in
 * chunks of any size, in order; the host does no per-packet work.  Packets (pack headers, system headers, PSM, padding,
 * private streams, PES) have variable lengths and may straddle chunks: every start code of a chunk is found, each
 * links to the one its packet's length reaches, and the chain from the position the previous chunk reached is found by
 * pointer jumping over those links; start codes inside payloads lie off the chain.  The chosen stream's PES headers
 * (MPEG-1: stuffing, STD buffer, PTS / DTS; MPEG-2: flags and header length) are parsed and their payloads appended
 * to the elementary stream, which sb_ps_finish decodes; messages about a frame name the file offset of the PES holding
 * its header.  Damage fails with SB_EINVAL naming the byte offset: a position the chain reaches that holds no start
 * code (a broken start code, a wrong length, bytes between packets), an invalid pack header, an invalid PES header of
 * the chosen stream.  A last PES cut by the file's end keeps its bytes and sets *cut; one cut inside its header is
 * dropped.  sb_ps_feed returns once the chunk is copied and scanned for start codes.  The sb_pcm outlives the sb_ps. */
int sb_ps_open(int32_t stream_id, int32_t substream_id, sb_ps** out);
int sb_ps_feed(sb_ps* ps, const void* host_chunk, int64_t nbytes, int64_t file_offset);
int sb_ps_finish(sb_ps* ps, int32_t* cut, sb_pcm** out);
int sb_ps_destroy(sb_ps* ps);

/* ---- Ogg FLAC (ABI version 15) -----------------------------------------------------------------------------------
 *
 * The FLAC stream with serial number `serial` of an Ogg file (the FLAC-to-Ogg mapping 1.0: a mapping header packet with
 * STREAMINFO, then `header_packets` metadata packets, then one FLAC frame per packet), demuxed on the GPU and decoded as
 * sb_flac_decode_frames decodes listed frames.  channels, bits (16 or 24) and rate come from STREAMINFO.  The file is
 * fed in chunks of any size, in order; the host does no per-page work.  Pages have variable lengths and may straddle
 * chunks: every capture pattern of a chunk is found, each links to the one its page's length reaches, and the chain
 * from the position the previous chunk reached is found by pointer jumping; capture patterns inside page bodies lie
 * off the chain.  Every page on the chain has its CRC-32 checked.  The chosen stream's pages are checked for sequence
 * numbers that follow each other and continuation flags that agree with the packet the page before left open, and
 * their bodies are appended to the stream whose packets sb_ogg_finish decodes; messages about a frame name the file
 * offset of the page where its packet starts.  Damage fails with SB_EINVAL naming the byte offset: a position the
 * chain reaches that holds no capture pattern, a version byte other than 0, a CRC mismatch, a sequence gap, a
 * continuation flag that contradicts the open packet, a page beginning a stream after the first data page (chained
 * Ogg).  A file cut inside a page drops that page and the packet it leaves open, and sets *cut.  sb_ogg_feed returns
 * once the chunk is copied and scanned for capture patterns.  The sb_pcm outlives the sb_ogg. */
int sb_ogg_open(uint32_t serial, int32_t channels, int32_t bits, int32_t rate, int32_t header_packets, sb_ogg** out);
int sb_ogg_feed(sb_ogg* ogg, const void* host_chunk, int64_t nbytes, int64_t file_offset);
int sb_ogg_finish(sb_ogg* ogg, int32_t* cut, sb_pcm** out);
int sb_ogg_destroy(sb_ogg* ogg);

/* ---- AVI (ABI version 18) ----------------------------------------------------------------------------------------
 *
 * One audio stream of an AVI file (OpenDML included), demuxed on the GPU: the payloads of its `NNwb` chunks (NN the
 * two decimal digits of stream_index, 0 to 99) in file order.  movi_extents[2 e], movi_extents[2 e + 1] are the file
 * offsets of the first chunk and the end of movi list e (sorted, none empty): the `LIST movi` of `RIFF AVI ` and of
 * each `RIFF AVIX`.  The file is fed in chunks of any size, in order; the host does no per-chunk work.  Chunks have
 * variable sizes and may straddle feeds: every chunk header of a feed (`NNwb`, `NNdc`, `NNdb`, `NNpc`, `NNtx`,
 * `ix##`, `JUNK`, `LIST rec `) is found, each links to the one its size (padded to even) reaches, `LIST rec ` to its
 * first child and a list's last chunk to the next list's first, and the chain from the position the previous feed
 * reached is found by pointer jumping; bytes the chain jumps over are not copied.  codec:
 *   SB_AVI_PCM  config[0..2] = channels (1 to 8), bits (16 or 24), rate: little-endian interleaved PCM, stored as
 *               sb_pcm_from_le stores it (24-bit samples by their top 16 bits); every chunk must hold whole sample
 *               frames;
 *   SB_AVI_MP2  the payloads are one MPEG audio stream, decoded as SB_TS_MP2 decodes a PID (config is not read);
 *               messages about a frame name the file offset of the chunk holding its header.
 * Damage fails with SB_EINVAL, "AVI chunk at byte offset N: ...", naming: a position the chain reaches that holds no
 * chunk header (a broken FOURCC, a wrong size, bytes between chunks), a chunk whose size runs past its movi list, a
 * PCM chunk that is not whole sample frames.  A last chunk cut by the file's end keeps the bytes there are and sets
 * *cut, as does a chain that stops short of the last list's end.  sb_avi_feed returns once the chunk is copied and
 * scanned for chunk headers.  The sb_pcm outlives the sb_avi. */
#define SB_AVI_PCM 0
#define SB_AVI_MP2 1
int sb_avi_open(int32_t stream_index, int32_t codec, const int32_t* config, const int64_t* movi_extents,
                int64_t n_extents, sb_avi** out);
int sb_avi_feed(sb_avi* avi, const void* host_chunk, int64_t nbytes, int64_t file_offset);
int sb_avi_finish(sb_avi* avi, int32_t* cut, sb_pcm** out);
int sb_avi_destroy(sb_avi* avi);

/* ---- multi-GPU: events shard across ranks (SURVEY.md 8e) ---------------- */

/* One process per GPU.  The library owns an NCCL communicator (libnccl is opened with dlopen on the first
 * of these calls; single-GPU users never need it).  The path has exactly two collectives, both outside the
 * kernels: a broadcast of the normalised streams (the reference's WavStream.data, wav.py:119-156, which every
 * rank needs) and an all-gather of the per-event (diff, idx) pairs find_substream returns (wav.py:188).
 * Rendezvous is the caller's business: rank 0 obtains SB_COMM_ID_BYTES opaque bytes from sb_comm_unique_id,
 * hands them to the other ranks by any means, then every rank calls sb_comm_init (collective). */
#define SB_COMM_ID_BYTES 128
int sb_comm_unique_id(void* id_out);
int sb_comm_init(const void* id, int world_size, int rank);
int sb_comm_destroy(void);
int sb_comm_world_size(void);                 /* 1 without a communicator */
int sb_comm_rank(void);
int sb_comm_nccl_version(void);               /* e.g. 22703; -1 if libnccl cannot be opened */
/* Broadcast `bytes` bytes of device memory in place from `root`.  Runs on the library's communication
 * stream, ordered behind everything the library stream has been given so far; `slot` (0..3) names the
 * completion event.  sb_comm_wait(slot) makes the library stream wait for that broadcast only, so the
 * broadcast of one stream overlaps the running sums and spectra of another. */
int sb_comm_broadcast(void* dev_buf, int64_t bytes, int root, int slot);
int sb_comm_wait(int slot);
/* All-gather on the library stream: every rank contributes bytes_per_rank bytes of device memory,
 * dev_recv receives world_size * bytes_per_rank bytes in rank order. */
int sb_comm_all_gather(const void* dev_send, void* dev_recv, int64_t bytes_per_rank);
/* Blocking helpers for measurement: element-wise maximum over ranks of up to 32 host floats (device
 * times are reported as the maximum over ranks), and a barrier that returns once every rank's
 * library and communication streams have drained. */
int sb_comm_max_f32(float* host_inout, int count);
int sb_comm_barrier(void);

/* ---- measurement ------------------------------------------------------- */

/* Device timer on the library stream (CUDA events). */
int sb_timer_start(void);
int sb_timer_stop(float* ms_out);
/* Per-kernel accounting: when enabled every kernel class is bracketed by CUDA
 * events on the library stream; sb_profile_get returns accumulated device ms
 * and launch count for a kernel class name (see DESIGN.md), sb_profile_names
 * a comma-separated list. Costs a little throughput while on. */
int sb_profile_enable(int on);
int sb_profile_reset(void);
int sb_profile_get(const char* name, double* ms_out, int64_t* launches_out);
const char* sb_profile_names(void);
/* Total kernels launched by this library since sb_init (or last reset). */
int64_t sb_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* SUSHI_B200_H */
