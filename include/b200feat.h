/*
 * b200feat — C ABI of the H100-native (sm_90a) batched Kaldi-style feature extractor.
 *
 * This header is the drop-in boundary for the ONE hot path this repository replaces:
 * lhotse's `FeatureExtractor.extract / extract_batch` for the Kaldi-compatible extractors
 * (reference citations are relative to the reference lhotse tree):
 *
 *   - lhotse/features/base.py:37-222          FeatureExtractor ABC (extract, extract_batch)
 *   - lhotse/features/kaldi/extractors.py:67  Fbank        (.extract :92, .extract_batch :117)
 *   - lhotse/features/kaldi/extractors.py:201 Mfcc         (.extract :222, .extract_batch :244)
 *   - lhotse/features/kaldi/extractors.py:297 Spectrogram  (.extract :318)
 *   - lhotse/features/kaldi/extractors.py:407 LogSpectrogram (.extract :428)
 *   - lhotse/features/kaldi/extractors.py:485 _extract_batch (pad, forward, trim)
 *   - lhotse/features/whisper_fbank.py:16-84  log_mel_spectrogram, :103 WhisperFbank (.extract :138)
 *   - lhotse/features/librosa_fbank.py:64-135 logmelfilterbank, :139 LibrosaFbank (.extract :157)
 *   - lhotse/features/kaldi/layers.py:151-186, :309-320, :392-402, :461-473, :565-578, :708-724
 *     (the arithmetic), :727-772 (framing), lhotse/utils.py:424-434 (frame-count contract)
 *
 * The reference is pure Python and has no FFI for this path; the binding a maintainer adds is
 * a `ctypes` stub inside a `FeatureExtractor` subclass — see INTEGRATION.md.  Everything here
 * is plain C: pointers, sizes, status codes.  No torch types, no C++ exceptions cross it.
 *
 * Ownership: the caller owns every sample/output/meta buffer; a handle owns only its immutable
 * constant tables (window, twiddles, sparse mel bank, DCT, lifter) on its device, plus — for
 * the `*_host` entry point only — a grow-only pinned/device staging ring.
 * Threading: a handle is immutable after create; `b200feat_extract` may be called concurrently
 * from several host threads on different streams.  `b200feat_extract_host` serialises on the
 * handle's staging ring.
 * Errors: every entry returns 0 on success or a negative B200FEAT_E* code; the message is
 * available from b200feat_last_error(handle) (or b200feat_global_error() when no handle exists).
 */
#ifndef B200FEAT_H_
#define B200FEAT_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200FEAT_ABI_VERSION 1

/* status codes */
#define B200FEAT_OK 0
#define B200FEAT_EINVAL (-1)      /* bad argument / inconsistent plan */
#define B200FEAT_EUNSUPPORTED (-2) /* plan not supported by any kernel */
#define B200FEAT_ECUDA (-3)       /* CUDA runtime error (message has the cudaError string) */
#define B200FEAT_ENODEVICE (-4)   /* no CUDA device / not an sm_90 part */
#define B200FEAT_ESHORT (-5)      /* a cut is too short to be framed (reference raises too) */

/* feature kinds — which reference module the plan mirrors */
#define B200FEAT_FBANK 0           /* Wav2LogFilterBank, layers.py:476 */
#define B200FEAT_MFCC 1            /* Wav2MFCC, layers.py:581 */
#define B200FEAT_SPECTROGRAM 2     /* Wav2Spec, layers.py:336 */
#define B200FEAT_LOG_SPECTROGRAM 3 /* Wav2LogSpec, layers.py:405 */
#define B200FEAT_WHISPER_FBANK 4   /* WhisperFbank / log_mel_spectrogram, lhotse/features/whisper_fbank.py:16-84:
                                      torch.stft(center=True) framing, log10(max(mel, mel_floor)), clamp to the cut's
                                      maximum - 8, (x + 4) / 4; rows beyond the stft's n/S frames are 0 (:73-80).
                                      Two launches per batch: the fused kernel (+ per-cut max) and a normalise pass. */

#define B200FEAT_LOG10_FBANK 5     /* LibrosaFbank / logmelfilterbank, lhotse/features/librosa_fbank.py:64-135: centred STFT
                                      (librosa.stft, pad_mode="reflect"), |X| (use_fft_mag) or |X|^2, mel, log10(max(., mel_floor));
                                      rows = compute_num_frames (:128-134).  One launch, any fast kernel. */

/* sample dtypes accepted by the kernels */
#define B200FEAT_F32 0 /* float32 in [-1, 1] — what lhotse hands to extract() */
#define B200FEAT_I16 1 /* int16 PCM; converted as x/32768 on load (libsndfile convention) */

/* output layouts */
#define B200FEAT_OUT_PACKED 0 /* (sum_i T_i, F) rows of cut i start at row_off[i] */
#define B200FEAT_OUT_PADDED 1 /* (B, T_max, F), rows >= T_i filled with pad_value
                                 (= collate_matrices(padding_value=LOG_EPSILON), collation.py:506) */

/* log-energy conventions (SURVEY.md §8a "semantic differences") */
#define B200FEAT_ENERGY_LHOTSE 0 /* max(log(sum + 1e-15), log(floor)) iff floor > 0; layers.py:859-870 */
#define B200FEAT_ENERGY_KALDI 1  /* max(log(max(sum, eps32)), log(floor)) iff floor != 0; torchaudio kaldi.py:116-122 */

/* framing / padding conventions (b200feat_plan_desc.pad_mode) */
#define B200FEAT_PAD_KALDI 0  /* lhotse/Kaldi: frame t starts at t*S - (L-S)/2, edges mirrored WITH the edge sample
                                 (x[-1] = x[0]); T = (n + S/2) / S; layers.py:753-772 */
#define B200FEAT_PAD_CENTER 1 /* torch.stft(center=True, pad_mode="reflect"): frame t starts at t*S - N/2, edges mirrored
                                 WITHOUT the edge sample (x[-1] = x[1]); needs n > N/2; whisper_fbank.py:62 */

/* kernel selection (b200feat_plan_desc.kernel) */
#define B200FEAT_KERNEL_AUTO 0
#define B200FEAT_KERNEL_GENERIC 1 /* any L/S/N, mixed-radix Stockham in shared memory */
#define B200FEAT_KERNEL_FAST 2    /* register-resident rFFT: N = 512 (radix 16x16, one frame per half-warp) or N = 256 (16x8, per quarter-warp) */
#define B200FEAT_KERNEL_TC 3      /* tensor cores: the N = 512 real DFT as two wgmma (3xTF32) GEMM stages, 8 frames per tile; fbank / mfcc */

typedef struct b200feat_plan_desc {
  int32_t struct_size;  /* sizeof(b200feat_plan_desc) — ABI guard */
  int32_t feature;      /* B200FEAT_FBANK ... */
  int32_t frame_length; /* L = floor(frame_length_s * sr), layers.py:114 */
  int32_t frame_shift;  /* S = floor(frame_shift_s * sr), layers.py:116 */
  int32_t fft_length;   /* N = next_pow2(L) or L, layers.py:264-265 */
  int32_t num_filters;  /* M (mel bins); 0 for the spectrogram kinds */
  int32_t num_ceps;     /* C (MFCC only) */
  int32_t snip_edges;   /* layers.py:747-751 */
  int32_t remove_dc_offset;
  int32_t use_energy;   /* 0 off; 1: fbank prepends the log-energy, spectrograms overwrite bin 0, mfcc replaces C0 (first column);
                           2 (fbank / mfcc): the same value in the LAST column (Kaldi's htk_compat layout) */
  int32_t raw_energy;   /* energy before (1) or after (0) pre-emphasis+window */
  int32_t use_fft_mag;  /* |X| instead of |X|^2 */
  int32_t energy_style; /* B200FEAT_ENERGY_* */
  int32_t use_lifter;   /* multiply cepstra by lifter[] */
  int32_t kernel;       /* B200FEAT_KERNEL_* */
  int32_t pad_mode;     /* B200FEAT_PAD_* (B200FEAT_PAD_CENTER goes with B200FEAT_WHISPER_FBANK and B200FEAT_LOG10_FBANK) */
  float preemph_coeff;  /* 0 disables, layers.py:165 */
  float energy_floor;   /* linear-domain floor (EPSILON = 1e-10 by default) */
  float mel_floor;      /* clamp before log for fbank/mfcc: finfo(float32).eps, layers.py:572 */
  float log_spec_eps;   /* log-spectrogram: eps >= 0 -> log(P + eps) (1e-15, layers.py:467); a negative value -f selects the
                           Kaldi / torchaudio form log(max(P, f)) (torchaudio/compliance/kaldi.py spectrogram, f = eps32) */
} b200feat_plan_desc;

typedef struct b200feat_handle b200feat_handle; /* opaque */

typedef struct b200feat_stats {
  int64_t calls;        /* extract launches since create */
  int64_t cuts;         /* cuts processed */
  int64_t frames;       /* feature rows produced */
  int64_t samples;      /* input samples consumed */
  int64_t kernel_launches; /* CUDA kernels launched by this handle */
} b200feat_stats;

/* Totals returned by b200feat_plan_batch. */
typedef struct b200feat_batch_totals {
  int64_t total_rows;    /* sum_i T_i (packed) */
  int64_t max_frames;    /* T_max */
  int64_t total_tiles;   /* work items of the selected kernel */
  int64_t span_samples;  /* elements the sample buffer must hold (last offset + last length) */
  int64_t out_floats;    /* floats the output buffer must hold for the chosen out_mode; for B200FEAT_WHISPER_FBANK this
                            includes B trailing scratch floats (the per-cut maxima) after the feature rows */
  int64_t meta_words;    /* int64 words of meta actually written (what must reach the device) */
} b200feat_batch_totals;

int b200feat_version(void);
const char *b200feat_global_error(void);

/*
 * Creates a handle on CUDA device `device`, uploading the constant tables.
 *   window   : L floats                    (create_frame_window, layers.py:921-940)
 *   mel_bank : K x M floats, row-major, K = N/2+1   (`_fb`, layers.py:541-563); NULL if M == 0
 *   dct      : M x C floats, row-major     (`_dct`, layers.py:697-706); NULL unless MFCC
 *   lifter   : C floats                    (`_lifter`, layers.py:681-695); NULL unless use_lifter
 * Tables are taken from the caller so that they are bit-identical to the reference's
 * float32 op sequence (and identical on every rank after an NCCL broadcast).
 */
int b200feat_create(const b200feat_plan_desc *desc, const float *window, const float *mel_bank,
                    const float *dct, const float *lifter, int device, b200feat_handle **out);
void b200feat_destroy(b200feat_handle *h);
const char *b200feat_last_error(const b200feat_handle *h);

/* T for a cut of n samples (layers.py:747-753); B200FEAT_ESHORT if it cannot be framed
 * (n too short for a single reflection — the reference raises on those, see SURVEY.md §7). */
int64_t b200feat_num_frames(const b200feat_handle *h, int64_t num_samples);
/* The same integer contract without a handle (and without a GPU): rows a cut of `num_samples` gets under `desc`, or
 * B200FEAT_ESHORT / B200FEAT_EINVAL.  Pure host arithmetic — lets build-time checks and CPU-only callers (manifest
 * validation: lhotse/qa.py:267-311 compares num_frames with compute_num_frames) agree with the kernels bit for bit. */
int64_t b200feat_desc_num_frames(const b200feat_plan_desc *desc, int64_t num_samples);
/* F: M (+1 with use_energy) for fbank, M for whisper-fbank / log10-fbank, C for mfcc, N/2+1 for the spectrogram kinds. */
int32_t b200feat_feature_dim(const b200feat_handle *h);
/* B200FEAT_KERNEL_GENERIC or B200FEAT_KERNEL_FAST — what AUTO resolved to. */
int32_t b200feat_kernel_kind(const b200feat_handle *h);
/* number of int64 words of the fixed part of the batch metadata for B cuts (4B + 2) */
int64_t b200feat_meta_words(int32_t batch);
/* exact number of int64 words b200feat_plan_batch writes for these cuts: the fixed part plus, for
 * tiled kernels, one int32 per tile mapping the tile to its cut (so that the kernel needs one load,
 * not a binary search, to locate its work).  Negative code on error (e.g. B200FEAT_ESHORT). */
int64_t b200feat_plan_words(const b200feat_handle *h, const int64_t *num_samples, int32_t batch,
                            int32_t out_mode);

/*
 * Host-side batch planning (pure integer work, no CUDA).
 *   num_samples[B]     : length of every cut
 *   sample_offsets[B]  : element offset of every cut in the sample buffer, or NULL to pack the
 *                        cuts back to back with each start aligned to `align` elements
 *   meta_host          : out, `meta_capacity` int64 words (>= b200feat_plan_words(...)); copy
 *                        totals->meta_words words verbatim to the device
 * Layout of meta: [0,B) sample offsets | [B,2B) lengths | [2B,3B+1) row prefix | [3B+1,4B+2) tile
 * prefix | int32 tile->cut table (tiled kernels only).
 */
int b200feat_plan_batch(const b200feat_handle *h, const int64_t *num_samples,
                        const int64_t *sample_offsets, int32_t batch, int32_t align,
                        int32_t out_mode, int64_t *meta_host, int64_t meta_capacity,
                        b200feat_batch_totals *totals);

/*
 * The hot call: device-resident ragged batch -> device-resident features.  Asynchronous on
 * `stream` (a cudaStream_t passed as void*; NULL = legacy default stream).
 *   samples_dev : float32 or int16 elements, addressed through meta's offsets
 *   meta_dev    : device copy of meta_host
 *   out_dev     : totals.out_floats floats, row-major (rows, F)
 */
int b200feat_extract(b200feat_handle *h, const void *samples_dev, int32_t sample_dtype,
                     const int64_t *meta_dev, int32_t batch, const b200feat_batch_totals *totals,
                     float *out_dev, int32_t out_mode, float pad_value, void *stream);

/*
 * Host-to-host convenience over the same kernels: what `FeatureExtractor.extract_batch` is for
 * numpy inputs.  Stages the ragged batch through the handle's pinned ring, overlaps H2D /
 * compute / D2H in chunks on internal streams, and blocks until `out_host` is complete.
 *   samples_host : the cuts back to back (element offsets = running sum of num_samples)
 *   out_host     : packed (sum T_i, F) or padded (B, T_max, F) floats
 */
int b200feat_extract_host(b200feat_handle *h, const void *samples_host, int32_t sample_dtype,
                          const int64_t *num_samples, int32_t batch, float *out_host,
                          int32_t out_mode, float pad_value);

/*
 * Same, with the cuts at caller-chosen element offsets inside `samples_host` (increasing, non-overlapping; NULL = back to
 * back as above).  Starting every cut on an even element keeps the kernels on their vector-load path: with back-to-back
 * staging every cut that follows an odd-length one is fetched tap by tap (correct, slower).
 */
int b200feat_extract_host_at(b200feat_handle *h, const void *samples_host, int32_t sample_dtype,
                             const int64_t *num_samples, const int64_t *sample_offsets, int32_t batch,
                             float *out_host, int32_t out_mode, float pad_value);

/*
 * Same, for cuts that live in SEPARATE host allocations (what `CutSet.compute_and_store_features_batch`, cut/set.py:2384, and
 * `OnTheFlyFeatures`, dataset/input_strategies.py:441, hand to `extract_batch`: a list of arrays): `cuts[i]` points at the
 * `num_samples[i]` samples of cut i.  The library gathers them into its pinned staging slots with a small thread pool
 * (non-temporal stores; B200FEAT_STAGING_THREADS, default 8), every cut on a 16-byte boundary, and overlaps the gather of chunk
 * c + 1 with the H2D / kernel / D2H of chunk c.  `out_host` as in b200feat_extract_host (pinned memory makes its copies async).
 */
int b200feat_extract_host_ptrs(b200feat_handle *h, const void *const *cuts, int32_t sample_dtype, const int64_t *num_samples,
                               int32_t batch, float *out_host, int32_t out_mode, float pad_value);

/* Read back a device-resident constant table (tests / NCCL-broadcast verification).
 * which: 0 window, 1 dense mel bank reconstructed from the sparse form (K x M), 2 dct, 3 lifter,
 * 4 twiddles (interleaved re,im). Returns the number of floats written or a negative code. */
int64_t b200feat_get_table(b200feat_handle *h, int32_t which, float *out, int64_t capacity);

/*
 * Optional per-column affine fused into every kernel's epilogue: each stored value v of output column c (and the padding
 * value of B200FEAT_OUT_PADDED rows) becomes v * scale[c] + shift[c].  With scale = 1 / std and shift = -mean / std this is
 * lhotse's GlobalMVN (lhotse/dataset/signal_transforms.py:16-58: (features - norm_means) / norm_stds on the collated batch)
 * without a second pass over the features.  `scale` / `shift`: F host floats each (copied); NULL, NULL switches it off.
 * Not available for B200FEAT_WHISPER_FBANK.  Call it while no extraction of this handle is in flight.
 */
int b200feat_set_output_affine(b200feat_handle *h, const float *scale, const float *shift);

int b200feat_get_stats(const b200feat_handle *h, b200feat_stats *out);

/*
 * FLAC (RFC 9639) on the GPU: 16-bit streams, 1-8 channels, every subframe type, both Rice methods, fixed and variable
 * blocking.  The host indexes a file once (pure host work, no device); the device decodes one frame per job into an int16
 * ragged buffer that b200feat_extract takes as B200FEAT_I16.
 */
typedef struct b200feat_flac_stream {
  int32_t struct_size;       /* sizeof(b200feat_flac_stream) — ABI guard */
  int32_t sample_rate, channels, bits_per_sample;
  int32_t min_block_size, max_block_size;
  int32_t variable_blocking; /* 1: frame headers carry the first sample number, 0: the frame number */
  int32_t reserved;
  int64_t total_samples;     /* per channel; 0 = unknown */
  int64_t audio_offset;      /* byte offset of the first frame */
  uint8_t md5[16];           /* MD5 of the interleaved little-endian samples */
} b200feat_flac_stream;

typedef struct b200feat_flac_frame {
  int64_t byte_offset, first_sample;
  int32_t block_size, byte_length; /* the last frame runs to the end of the file */
} b200feat_flac_frame;

/* Parses STREAMINFO and finds every frame of a whole file held in memory.  A sync candidate is a frame only when its
 * reserved bits are zero, its CRC-8 holds, its frame / first-sample number is the next one expected, and its block size and
 * channel count agree with STREAMINFO.  Returns the frame count (frames beyond `capacity` are counted, not written) or a
 * negative B200FEAT_E* code. */
int64_t b200feat_flac_index(const uint8_t *file, int64_t nbytes, b200feat_flac_stream *info, b200feat_flac_frame *frames,
                            int64_t capacity);

/* One job = one FLAC frame of one cut: samples [skip, skip + count) of channel `want_channel` go to
 * out_dev[dst_elem, dst_elem + count).  A job of a multi-channel stream gets `count` int32 of scratch at element
 * `scratch_elem` (decorrelated stereo needs the other channel at the same index); -1 for mono. */
typedef struct b200feat_flac_job {
  int64_t src_byte;       /* first byte of the frame in bytes_dev */
  int64_t dst_elem;
  int64_t scratch_elem;
  int64_t coded_number;   /* frame number (fixed blocking) or first sample number (variable blocking) the header must carry */
  int32_t byte_length, block_size, channels, want_channel, skip, count, variable_blocking, reserved;
} b200feat_flac_job;

/* per-job status written by b200feat_flac_decode */
#define B200FEAT_FLAC_OK 0
#define B200FEAT_FLAC_EJOB 1       /* the job itself is inconsistent (window, channel, scratch, lengths) */
#define B200FEAT_FLAC_EHEADER 2    /* sync, reserved bits, CRC-8, or a header that disagrees with the job */
#define B200FEAT_FLAC_ECRC 3       /* CRC-16 of the frame */
#define B200FEAT_FLAC_ERESERVED 4  /* reserved subframe type or residual method, non-zero subframe pad bit */
#define B200FEAT_FLAC_EPRECISION 5 /* LPC coefficient precision code 1111 */
#define B200FEAT_FLAC_ESHIFT 6     /* negative LPC shift */
#define B200FEAT_FLAC_EPARTITION 7 /* partition order / predictor order that does not fit the block */
#define B200FEAT_FLAC_ERANGE 8     /* a sample outside its subframe's width or outside int16, wasted bits >= width */
#define B200FEAT_FLAC_ETRUNCATED 9 /* the subframes run past the frame's bytes */
#define B200FEAT_FLAC_ELENGTH 10   /* the subframes end before the frame's CRC-16 */

/* Device-resident and asynchronous on `stream`: decodes `njobs` jobs out of bytes_dev into out_dev (`out_elems` int16) and
 * writes status_dev[j] (B200FEAT_FLAC_*).  Malformed frames yield a status, never an access outside the job's byte range or
 * output window. */
int b200feat_flac_decode(const uint8_t *bytes_dev, const b200feat_flac_job *jobs_dev, int32_t njobs, int16_t *out_dev,
                         int64_t out_elems, int32_t *status_dev, void *scratch_dev, int64_t scratch_bytes, void *stream);

/*
 * Audio-domain mixing of mono int16 tracks on the GPU: what lhotse's MixedCut.load_audio() computes under NumPy >= 2, bit
 * for bit (DESIGN.md §3.1h).  The tracks are samples of two int16 device buffers (e.g. a PCM16 batch and a FLAC decode);
 * every cut's mix is written as float32 into a ragged output buffer that b200feat_extract takes as B200FEAT_F32.
 */
#define B200FEAT_MIX_SRC_F32 2      /* b200feat_mix_track.source: the float32 track buffer of b200feat_mix_ex (read as is) */
#define B200FEAT_MIX_ROLE_MIXED 0   /* the track is part of the mix (the cut's first such track is the mixer's base) */
#define B200FEAT_MIX_ROLE_ENERGY 1  /* a muted SNR reference: its energy sets the gains, its samples are not mixed */
#define B200FEAT_MIX_F32 0          /* cut mode: a float32 mix */
#define B200FEAT_MIX_SCALED_FIRST 1 /* cut mode: the first track carries an SNR against another reference; when both energies
                                       are positive it is scaled in float64 and the whole mix is float64 */

typedef struct b200feat_mix_track {
  int32_t struct_size;   /* sizeof(b200feat_mix_track) — ABI guard, in every record */
  int32_t source;        /* 0: src0, 1: src1, -1: padding (zeros), B200FEAT_MIX_SRC_F32: src2 (b200feat_mix_ex only) */
  int64_t src_elem;      /* first sample of the track in its source buffer */
  int64_t num_samples;   /* track length */
  int64_t mix_offset;    /* first sample of the track in the mix */
  double snr_factor;     /* 10 ** (-snr / 10) as the host evaluates it; NaN: the track has no SNR */
  int32_t cut;           /* index of the cut the track belongs to */
  int32_t role;          /* B200FEAT_MIX_ROLE_* */
} b200feat_mix_track;

typedef struct b200feat_mix_cut {
  int32_t struct_size;   /* sizeof(b200feat_mix_cut) */
  int32_t mode;          /* B200FEAT_MIX_F32 | B200FEAT_MIX_SCALED_FIRST */
  int64_t out_elem;      /* first output element of the cut */
  int64_t mix_len;       /* max(offset + length) over the mixed tracks */
  int64_t target_len;    /* the cut's length: the mix is trimmed, or reflect-padded by at most mix_len - 1 samples */
  int32_t first_track;   /* the cut's tracks are [first_track, first_track + num_tracks) of the track table, in track order */
  int32_t num_tracks;
  int32_t ref_track;     /* the SNR reference, relative to first_track */
  int32_t reserved;
} b200feat_mix_cut;

/* Device scratch b200feat_mix needs for `ntracks` tracks and `ncuts` cuts. */
int64_t b200feat_mix_work_bytes(int32_t ntracks, int32_t ncuts);

/* Checks the host tables (every track inside its source buffer, every cut inside the output, source and reference indices),
 * copies them to `work_dev` and launches the energy and mix kernels, asynchronously on `stream`.  The tables may be pinned:
 * they are read by the copy on `stream`, so they must stay unchanged until it has run.  Errors are reported through `h`
 * (b200feat_last_error) when it is not NULL, and through b200feat_global_error. */
int b200feat_mix(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev, int64_t src1_elems,
                 const b200feat_mix_track *tracks, int32_t ntracks, const b200feat_mix_cut *cuts, int32_t ncuts,
                 float *out_dev, int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream);

/* b200feat_mix with a third, float32 source: tracks whose `source` is B200FEAT_MIX_SRC_F32 read `src2_dev` (for example
 * perturbed tracks that b200feat_resample wrote), their samples taken as they are instead of q / 32768.  The same checks,
 * plus: such a track lies inside src2 and src2 is present.  b200feat_mix is this call with no src2. */
int b200feat_mix_ex(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev, int64_t src1_elems,
                    const float *src2_dev, int64_t src2_elems, const b200feat_mix_track *tracks, int32_t ntracks,
                    const b200feat_mix_cut *cuts, int32_t ncuts, float *out_dev, int64_t out_elems, void *work_dev,
                    int64_t work_bytes, void *stream);

/*
 * Resampling and volume scaling of mono audio on the GPU: lhotse's Speed, Resample and Volume transforms as its CPU route
 * computes them when torch runs the resampling conv1d through oneDNN, bit for bit (DESIGN.md §3.1i).  A cut's transform
 * chain is a list of stages; stage 0 reads one of two int16 device buffers (e.g. a PCM16 batch and a FLAC decode), later
 * stages read a float32 intermediate buffer, and the last stage writes the cut's float32 samples into a ragged output buffer
 * that b200feat_extract takes as B200FEAT_F32.
 */
#define B200FEAT_RESAMPLE_SRC0 0    /* stage source: src0 (int16) */
#define B200FEAT_RESAMPLE_SRC1 1    /* stage source: src1 (int16) */
#define B200FEAT_RESAMPLE_MID 2     /* stage source: the float32 intermediate buffer */
#define B200FEAT_RESAMPLE_TO_MID 0  /* stage target: the float32 intermediate buffer */
#define B200FEAT_RESAMPLE_TO_OUT 1  /* stage target: the output buffer (the cut's final samples) */

typedef struct b200feat_resample_stage {
  int32_t struct_size;   /* sizeof(b200feat_resample_stage) — ABI guard, in every record */
  int32_t table;         /* id from b200feat_resample_table; -1: no resampling (the scales only) */
  int32_t source;        /* B200FEAT_RESAMPLE_SRC0 | _SRC1 | _MID */
  int32_t target;        /* B200FEAT_RESAMPLE_TO_MID | _TO_OUT */
  int32_t depth;         /* stages run in depth order (the records are sorted by it): depth d reads what depth d - 1 wrote */
  float scale_in;        /* every input sample is multiplied by it on load (a Volume before the resampler; 1: none) */
  float scale_out;       /* every output sample is multiplied by it before the store (a Volume after it; 1: none) */
  int32_t reserved;
  int64_t in_elem;       /* first input sample in the source buffer */
  int64_t in_len;        /* L, at least 1 */
  int64_t out_elem;      /* first output sample in the target buffer */
  int64_t out_len;       /* for a table of the pair O -> N: min(ceil(f32(N * L / O)), N * (L / O + 1)), the quotient
                            evaluated in double and rounded to float as lhotse's torch.as_tensor does; L without a table */
  int64_t target_len;    /* samples written: out_len, or (target _TO_OUT only) fewer (trimmed) or at most out_len - 1 more
                            (np.pad(mode="reflect")) */
} b200feat_resample_stage;

/* Registers the float32 table kernel[rows][taps] (rows = N, taps = 2 * width + O for the pair orig -> new reduced by their
 * gcd to O -> N) on the current device and returns its id in *table_id.  Tables are kept per (device, orig, new) for the
 * life of the process: when the pair is known on this device the stored table's id is returned and `kernel` is not read.
 * B200FEAT_EINVAL for inconsistent sizes, or a table with taps + O > 8192 or more than 2^22 entries. */
int b200feat_resample_table(b200feat_handle *h, int32_t orig, int32_t new_rate, const float *kernel, int32_t rows, int32_t taps,
                            int32_t width, int32_t *table_id);

/* Device scratch b200feat_resample needs for `nstages` stages. */
int64_t b200feat_resample_work_bytes(int32_t nstages);

/* Checks the host stage records (every read inside its source, every write inside its target, table ids of this device,
 * out_len as above, reflect padding shorter than the stage output, depth order), copies them to `work_dev`
 * and launches one kernel per depth, asynchronously on `stream`.  Errors are reported through `h` (b200feat_last_error) when
 * it is not NULL, and through b200feat_global_error. */
int b200feat_resample(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev,
                      int64_t src1_elems, float *mid_dev, int64_t mid_elems, const b200feat_resample_stage *stages,
                      int32_t nstages, float *out_dev, int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream);

/*
 * Reverberation of mono float32 audio with room impulse responses on the GPU: lhotse's ReverbWithImpulseResponse with a
 * recorded mono RIR (shift output, normalize_output optional), within a float32 tolerance of a float64 convolution
 * (DESIGN.md §3.1j).  The RIRs are int16 samples of two device buffers (e.g. a PCM16 batch and a FLAC decode), taken as
 * f32(q / 32768) * 2^-15 as lhotse scales them; the inputs are float32 samples of one buffer (e.g. what b200feat_resample or
 * b200feat_mix_ex wrote); every cut's result is written as float32 into a ragged output buffer that b200feat_extract takes as
 * B200FEAT_F32.
 */
#define B200FEAT_REVERB_MAX_RIR 65536  /* the longest RIR, in samples */

typedef struct b200feat_reverb_rir {
  int32_t struct_size;   /* sizeof(b200feat_reverb_rir) — ABI guard, in every record */
  int32_t source;        /* 0: src0, 1: src1 */
  int64_t src_elem;      /* first RIR sample in its source buffer */
  int64_t num_samples;   /* R, 1 <= R <= B200FEAT_REVERB_MAX_RIR */
} b200feat_reverb_rir;

typedef struct b200feat_reverb_cut {
  int32_t struct_size;   /* sizeof(b200feat_reverb_cut) */
  int32_t rir;           /* index into the RIR table */
  int32_t normalize;     /* 1: scale the result to the input's power (lhotse's normalize_output), 0: leave it */
  int32_t reserved;
  int64_t in_elem;       /* first input sample in the input buffer */
  int64_t in_len;        /* N, at least 1: the output of the reverb has N samples too */
  int64_t out_elem;      /* first output sample in the output buffer */
  int64_t target_len;    /* samples written: N, fewer (trimmed) or at most N - 1 more (np.pad(mode="reflect")) */
} b200feat_reverb_cut;
/* The input and output buffers may be one allocation, but no cut's output window [out_elem, out_elem + target_len) may
 * overlap any cut's input window [in_elem, in_elem + in_len) in memory: b200feat_reverb refuses such tables. */

/* Device scratch b200feat_reverb needs for these tables (0 when a count is negative). */
int64_t b200feat_reverb_work_bytes(const b200feat_reverb_rir *rirs, int32_t nrirs, const b200feat_reverb_cut *cuts, int32_t ncuts);

/* Checks the host tables (every read inside its source, every write inside the output, RIR indices, 1 <= R <= the cap,
 * reflect padding shorter than the signal), copies what the kernels read to `work_dev` and launches the RIR spectra,
 * convolution, gain and output kernels, asynchronously on `stream`.  Output windows must not overlap input windows (above).  Results are identical from run to run.  Errors are
 * reported through `h` (b200feat_last_error) when it is not NULL, and through b200feat_global_error. */
int b200feat_reverb(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev, int64_t src1_elems,
                    const float *in_dev, int64_t in_elems, const b200feat_reverb_rir *rirs, int32_t nrirs,
                    const b200feat_reverb_cut *cuts, int32_t ncuts, float *out_dev, int64_t out_elems, void *work_dev,
                    int64_t work_bytes, void *stream);

#define B200FEAT_REVERB_RIR_F32 2  /* b200feat_reverb_rir.source of b200feat_reverb_ex: the float32 RIR buffer */

/* b200feat_reverb with a third RIR source: records whose `source` is B200FEAT_REVERB_RIR_F32 read float32 samples of
 * `rir32_dev` (for example RIRs that b200feat_rir_generate and b200feat_resample wrote), scaled by 2^-15 as lhotse scales
 * them; the shift is the first index of their maximum.  The same checks, plus: such an RIR lies inside rir32.
 * b200feat_reverb is this call with no rir32.  The work buffer is b200feat_reverb_work_bytes of the same tables. */
int b200feat_reverb_ex(b200feat_handle *h, const int16_t *src0_dev, int64_t src0_elems, const int16_t *src1_dev,
                       int64_t src1_elems, const float *rir32_dev, int64_t rir32_elems, const float *in_dev, int64_t in_elems,
                       const b200feat_reverb_rir *rirs, int32_t nrirs, const b200feat_reverb_cut *cuts, int32_t ncuts,
                       float *out_dev, int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream);

/*
 * Single-channel WPE dereverberation on the GPU: lhotse's DereverbWPE (torch.stft with a centred, reflect-padded frame and
 * the periodic Blackman window, nara_wpe's wpe_v8, torch.istft, then the cut's length fix), within a float32 tolerance of a
 * float64 restatement (DESIGN.md §3.1q).  The inputs are float32 samples of one buffer (e.g. what b200feat_resample or
 * b200feat_reverb wrote); every cut's result is written as float32 into a ragged output buffer that b200feat_extract takes
 * as B200FEAT_F32.  A cut of L samples has T = 1 + L / 128 frames and dereverberates to 128 (T - 1) = 128 (L / 128) samples.
 */
#define B200FEAT_WPE_MAX_TAPS 16      /* the most filter taps */
#define B200FEAT_WPE_MAX_FRAMES 8192  /* the most frames of one cut (L <= 1048575: 65.5 s at 16 kHz) */
#define B200FEAT_WPE_FULL 0           /* b200feat_wpe_params.statistics_mode: statistics over every frame */
#define B200FEAT_WPE_VALID 1          /* ... over the frames t >= delay + taps - 1 */

typedef struct b200feat_wpe_params {
  int32_t struct_size;      /* sizeof(b200feat_wpe_params) — ABI guard */
  int32_t n_fft;            /* 512: the only transform size */
  int32_t hop;              /* 128: the only hop */
  int32_t taps;             /* 1 .. B200FEAT_WPE_MAX_TAPS (lhotse: 10) */
  int32_t delay;            /* >= 0 (lhotse: 3) */
  int32_t iterations;       /* 0 .. 64 (lhotse: 3; 0 leaves the spectra as they are) */
  int32_t statistics_mode;  /* B200FEAT_WPE_FULL | B200FEAT_WPE_VALID */
  int32_t reserved;
} b200feat_wpe_params;

typedef struct b200feat_wpe_cut {
  int32_t struct_size;   /* sizeof(b200feat_wpe_cut) — ABI guard, in every record */
  int32_t reserved;
  int64_t in_elem;       /* first input sample in the input buffer */
  int64_t in_len;        /* L: more than 256 (the reflect pad), 1 + L / 128 >= taps + delay, at most B200FEAT_WPE_MAX_FRAMES frames */
  int64_t out_elem;      /* first output sample in the output buffer */
  int64_t target_len;    /* samples written: 128 (L / 128), fewer (trimmed) or at most 128 (L / 128) - 1 more (np.pad(mode="reflect")) */
} b200feat_wpe_cut;
/* No cut's output window [out_elem, out_elem + target_len) may overlap any cut's input window [in_elem, in_elem + in_len)
 * in memory: b200feat_wpe refuses such tables, and leaves the input as it was. */

/* Device scratch b200feat_wpe needs for these cuts (0 when the count is negative): the cuts' spectra, 257 x T complex64 per
 * cut (about 16 bytes per input sample), plus a few KB of tables. */
int64_t b200feat_wpe_work_bytes(const b200feat_wpe_cut *cuts, int32_t ncuts);

/* Checks the parameters (n_fft and hop other than 512 and 128: B200FEAT_EUNSUPPORTED; taps, delay, iterations and
 * statistics_mode outside their ranges: B200FEAT_EINVAL) and the cut table (a cut too short for the reflect pad or with
 * fewer than taps + delay frames: B200FEAT_ESHORT; more than B200FEAT_WPE_MAX_FRAMES frames, a read outside the input, a
 * write outside the output, reflect padding longer than the signal, an output overlapping an input: B200FEAT_EINVAL), copies
 * the tables and the host `window` (n_fft floats: torch.blackman_window(512)'s float32 values) to `work_dev` and launches
 * the STFT, per-bin and iSTFT kernels, asynchronously on `stream`.  No atomics: results are identical from run to run, and
 * a cut's output does not depend on the other cuts of the call.  Errors are reported through `h` (b200feat_last_error)
 * when it is not NULL, and through b200feat_global_error. */
int b200feat_wpe(b200feat_handle *h, const float *in_dev, int64_t in_elems, const b200feat_wpe_cut *cuts, int32_t ncuts,
                 const b200feat_wpe_params *params, const float *window, float *out_dev, int64_t out_elems, void *work_dev,
                 int64_t work_bytes, void *stream);

/*
 * lhotse's FastRandomRIRGenerator (one source) on the GPU, from draws made on the host (DESIGN.md §3.1l): the Dirac comb at
 * 64 x sr, its 8 -> 1 resampling and torchaudio's 80 Hz highpass biquad, written as float32 at 8 x sr.  b200feat_resample
 * with the same 8 -> 1 table then gives the RIR at sr.  Results are identical from run to run.
 */
#define B200FEAT_RIRGEN_TAPS 106  /* the 8 -> 1 resampler table: 2 * 49 + 8 taps */

typedef struct b200feat_rir_gen {
  int32_t struct_size;   /* sizeof(b200feat_rir_gen) — ABI guard, in every record */
  int32_t sampling_rate; /* the generator's sr, 1 .. 192000: 2 sr image sources, a comb at 64 sr */
  double t60;            /* room_rng's T60 draw, > 0 */
  double r;              /* room_rng's R draw */
  double d0;             /* source_rng's distance draw, > 0 and below 340 t60 (f32(340 t60 / d0 - 1) > 0: the last image
                            ratio; lhotse's draws always are, d0 <= 12 < 34 <= 340 t60), or the record is refused */
  double tau;            /* the generator's tau */
  float b0, b1, b2, a1, a2;  /* highpass_biquad(., 8 sr, 80)'s coefficients divided by a0, as torchaudio's lfilter takes them */
  int32_t reserved;
  int64_t cdf_elem;      /* first of the 2 sr entries of the normalised cumulative distribution (float32, last one 1) */
  int64_t draw_elem;     /* first of the 2 sr multinomial uniforms in the draws buffer; the 2 sr perturbations follow */
  int64_t comb_len;      /* L = ceil(64 sr T60) as lhotse computes it, 1 .. 2^31 - 1 */
  int64_t out_elem;      /* first output sample */
  int64_t out_len;       /* min(ceil(f32(L / 8)), L / 8 + 1): what lhotse's first resampler keeps */
} b200feat_rir_gen;

/* Device scratch b200feat_rir_generate needs for these records (0 when the count is negative or a record is malformed). */
int64_t b200feat_rir_generate_work_bytes(const b200feat_rir_gen *rirs, int32_t nrirs);

/* Checks the records (every read inside its buffer, every output inside `out_dev` and disjoint from the others, the lengths
 * as above), copies them and the host table `table` (B200FEAT_RIRGEN_TAPS floats, lhotse's 8 -> 1 resampler) to `work_dev`
 * and launches the entry kernel, the segmented sort, the window kernel and the biquad kernel, asynchronously on `stream`.
 * Errors are reported through `h` (b200feat_last_error) when it is not NULL, and through b200feat_global_error. */
int b200feat_rir_generate(b200feat_handle *h, const double *draws_dev, int64_t draws_elems, const float *cdf_dev,
                          int64_t cdf_elems, const float *table, const b200feat_rir_gen *rirs, int32_t nrirs, float *out_dev,
                          int64_t out_elems, void *work_dev, int64_t work_bytes, void *stream);

/*
 * SpecAugment on a padded (B, T, F) float32 feature batch on the GPU: what lhotse's SpecAugment.forward computes from the
 * same random draws (DESIGN.md §3.1k).  The host draws the numbers and hands over two tables: the time warps (bicubic along
 * time, within a float32 tolerance of lhotse's F.interpolate) and the mask rectangles, which are filled with the mean of the
 * sequence's whole warped (T, F) matrix.  Everything outside warped segments and masks is copied bit for bit.
 */
#define B200FEAT_SPECAUG_TIME 0     /* b200feat_specaug_mask.axis: frames [start, end) of every feature bin */
#define B200FEAT_SPECAUG_FEATURE 1  /* feature bins [start, end) of every frame */

typedef struct b200feat_specaug_warp {
  int32_t struct_size;   /* sizeof(b200feat_specaug_warp) — ABI guard, in every record */
  int32_t seq;           /* sequence index, in [0, B) */
  int32_t start;         /* first frame of the segment; the segments of one sequence must not overlap */
  int32_t len;           /* its frames: [start, start + len) inside [0, T) */
  int32_t center;        /* 0 < center < len: input frames [0, center) of the segment ... */
  int32_t warped;        /* 0 < warped < len: ... become its output frames [0, warped), the rest the rest */
} b200feat_specaug_warp;

typedef struct b200feat_specaug_mask {
  int32_t struct_size;   /* sizeof(b200feat_specaug_mask) */
  int32_t seq;           /* sequence index, in [0, B) */
  int32_t axis;          /* B200FEAT_SPECAUG_TIME | B200FEAT_SPECAUG_FEATURE */
  int32_t start;         /* 0 <= start <= end <= T (time) or F (feature) */
  int32_t end;
  int32_t reserved;
} b200feat_specaug_mask;

/* Device scratch b200feat_specaug needs (0 when an argument is out of range). */
int64_t b200feat_specaug_work_bytes(int32_t B, int32_t T, int32_t F, int32_t nwarps, int32_t nmasks);

/* Checks the host tables (sequence indices, every segment inside [0, T) with 0 < center, warped < len, the segments of a
 * sequence disjoint, every rectangle inside its axis with start <= end, in_dev != out_dev, T * F < 2^31), copies them to
 * `work_dev` and launches the warp-and-copy, mean and mask-fill kernels, asynchronously on `stream`: three launches whatever
 * B is.  `in_dev` is read only; every element of `out_dev` is written.  Results are identical from run to run.  Errors are
 * reported through `h` (b200feat_last_error) when it is not NULL, and through b200feat_global_error. */
int b200feat_specaug(b200feat_handle *h, const float *in_dev, float *out_dev, int32_t B, int32_t T, int32_t F,
                     const b200feat_specaug_warp *warps, int32_t nwarps, const b200feat_specaug_mask *masks, int32_t nmasks,
                     void *work_dev, int64_t work_bytes, void *stream);

/*
 * Feature-domain mixing and right-padding collation of precomputed feature rows on the GPU: what lhotse's collate_features
 * computes for cuts whose features are stored (MixedCut.load_features with its FeatureMixer, PaddingCut constants, the
 * padding-only copy), within a float32 rounding of a float64 evaluation of the same tables (DESIGN.md §3.1m).  The stored
 * rows are float32 elements of one device buffer (row-major, F per row); the output is a padded (B, T_max, F) float32 batch.
 */
#define B200FEAT_FEATMIX_LOG 0       /* mix law: log(max(EPSILON, e^a + g e^b)), energy sum e^x, scale x + log g (Fbank family) */
#define B200FEAT_FEATMIX_LINEAR 1    /* mix law: a + g b, energy sum x, scale g x (Spectrogram) */
#define B200FEAT_FEATMIX_COPY 0      /* cut mode: its one track's rows as they are, then pad_value up to num_rows */
#define B200FEAT_FEATMIX_MIX 1       /* cut mode: FeatureMixer over its tracks, in track order */
#define B200FEAT_FEATMIX_MIXED 1     /* track flag: the track is part of the mix (the cut's first track is the mixer's base) */
#define B200FEAT_FEATMIX_ENERGY 2    /* track flag: the cut needs the track's energy (its SNR reference, a track with an SNR) */

typedef struct b200feat_featmix_track {
  int32_t struct_size;   /* sizeof(b200feat_featmix_track) — ABI guard, in every record */
  int32_t cut;           /* index of the cut the track belongs to */
  int32_t flags;         /* B200FEAT_FEATMIX_MIXED | B200FEAT_FEATMIX_ENERGY */
  int32_t stored_rows;   /* rows in the source buffer; 0: a constant track (every element is `value`) */
  int32_t num_rows;      /* rows the track has: stored_rows, or stored_rows + 1 (the last stored row repeated) */
  int32_t offset;        /* first mix row of the track (0 for the cut's first track) */
  float value;           /* the element value of a constant track (a PaddingCut's feat_value as float32) */
  int32_t reserved;
  int64_t src_elem;      /* first element of the stored rows in the source buffer */
  double snr_factor;     /* 10 ** (-snr / 10) as the host evaluates it; NaN: the track has no SNR */
} b200feat_featmix_track;

typedef struct b200feat_featmix_cut {
  int32_t struct_size;   /* sizeof(b200feat_featmix_cut) */
  int32_t mode;          /* B200FEAT_FEATMIX_COPY | B200FEAT_FEATMIX_MIX */
  int32_t law;           /* B200FEAT_FEATMIX_LOG | B200FEAT_FEATMIX_LINEAR (MIX cuts) */
  int32_t num_rows;      /* the cut's rows in the output, at most T_max; rows past it are the call's pad_value */
  int32_t mix_rows;      /* MIX: the mixer's rows (the base's, grown by every further track's offset + rows), within one
                            row of num_rows: trimmed, or the last mix row repeated */
  int32_t first_track;   /* the cut's tracks are [first_track, first_track + num_tracks) of the track table, in track order */
  int32_t num_tracks;    /* COPY: 1 */
  int32_t ref_track;     /* MIX: the SNR reference, relative to first_track */
  float pad_value;       /* COPY: the value of rows [track rows, num_rows) */
  int32_t reserved;
} b200feat_featmix_cut;

/* Device scratch b200feat_feature_mix needs for `ntracks` tracks and `ncuts` cuts (0 when a count is negative). */
int64_t b200feat_feature_mix_work_bytes(int32_t ntracks, int32_t ncuts);

/* Checks the host tables (every track inside the source buffer and linked to its cut, row counts, flags, law and mode codes,
 * mix_rows the end of the cut's mixed tracks, at most 65535 cuts), copies them to `work_dev` and launches the energy, gain
 * and output kernels, asynchronously on `stream`: three launches whatever the batch.  Every element of the
 * (ncuts, T_max, F) output `out_dev` is written.  Results are identical from run to run.  Errors are reported through `h`
 * (b200feat_last_error) when it is not NULL, and through b200feat_global_error. */
int b200feat_feature_mix(b200feat_handle *h, const float *src_dev, int64_t src_elems, const b200feat_featmix_track *tracks,
                         int32_t ntracks, const b200feat_featmix_cut *cuts, int32_t ncuts, int32_t F, float *out_dev,
                         int32_t T_max, float pad_value, void *work_dev, int64_t work_bytes, void *stream);

/*
 * Backward of the Kaldi-family kinds (B200FEAT_FBANK, _MFCC, _SPECTROGRAM, _LOG_SPECTROGRAM, Kaldi framing): the gradient of
 * a scalar loss with respect to the float32 samples, given its gradient with respect to the packed (sum T_i, F) rows that
 * b200feat_extract produced from the same samples (DESIGN.md §3.1n).  The frames are recomputed from the samples; nothing
 * of the forward is kept.
 */
/* Device scratch b200feat_backward (b200feat_whisper_backward for a whisper-fbank handle) needs for cuts of `num_samples`
 * (host array of B), or a negative B200FEAT_E* code (B200FEAT_ESHORT for a cut too short to be framed, B200FEAT_EINVAL for a
 * kind without a backward). */
int64_t b200feat_backward_work_bytes(b200feat_handle *h, const int64_t *num_samples, int32_t B);

/* `samples_dev` (B200FEAT_F32 only) holds cut i at element offsets[i] with num_samples[i] samples (host arrays); `grad_out_dev`
 * the (row_off[B], F) gradient of the features, cut i's rows at [row_off[i], row_off[i + 1]) (host array of B + 1 with
 * row_off[0] = 0 and each cut's frame count).  Writes the gradient of every sample [offsets[i], offsets[i] + num_samples[i])
 * of `grad_in_dev` (same layout as the samples; elements outside the cuts are not touched), asynchronously on `stream`: two
 * launches.  No atomics: results are identical from run to run, and a cut's gradient does not depend on the other cuts of the
 * call.  Errors are reported through `h` (b200feat_last_error). */
int b200feat_backward(b200feat_handle *h, const float *samples_dev, int32_t dt, const int64_t *num_samples, const int64_t *offsets,
                      int32_t B, const float *grad_out_dev, const int64_t *row_off, float *grad_in_dev, void *work_dev,
                      int64_t work_bytes, void *stream);

/*
 * Backward of whisper-fbank (DESIGN.md §3.1p).  Its forward clamps every log-mel value to its cut's maximum - 8, a cut-wide
 * decision a recomputation by another FFT cannot repeat bit for bit, so the backward reads the forward's own un-normalised
 * log-mel rows and maxima, which b200feat_extract_keep_raw keeps.
 */
/* b200feat_extract for a whisper-fbank handle and a batch planned with B200FEAT_OUT_PACKED, keeping what the backward
 * needs: the fused kernel writes the (total_rows, F) log-mel rows to `raw_dev`, followed by the B per-cut maxima
 * (`tot->out_floats` floats in all), and the normalise pass writes the features to `out_dev` ((total_rows, F) floats),
 * bitwise equal to b200feat_extract's.  Both buffers 16-byte aligned.  Two launches, asynchronous on `stream`. */
int b200feat_extract_keep_raw(b200feat_handle *h, const void *samples_dev, int32_t dt, const int64_t *meta_dev, int32_t B,
                              const b200feat_batch_totals *tot, float *out_dev, float *raw_dev, void *stream);

/* b200feat_backward for a whisper-fbank handle (whose b200feat_backward refuses and names this entry), with the forward's
 * log-mel rows `raw_dev` (laid out as grad_out_dev) and per-cut maxima `cut_max_dev` [B] from b200feat_extract_keep_raw.
 * b200feat_backward_work_bytes gives the scratch it needs.  The same argument checks (a cut of n <= fft_length / 2
 * samples: B200FEAT_ESHORT, as the forward; a row_off that does not match a cut's rows; samples other than
 * B200FEAT_F32), then three launches: a per-cut reduction, frames, combine.  No atomics: results are identical from run to
 * run, and a cut's gradient does not depend on the other cuts of the call.  The gradient of the extra zero row is ignored. */
int b200feat_whisper_backward(b200feat_handle *h, const float *samples_dev, int32_t dt, const int64_t *num_samples,
                              const int64_t *offsets, int32_t B, const float *grad_out_dev, const float *raw_dev,
                              const float *cut_max_dev, const int64_t *row_off, float *grad_in_dev, void *work_dev,
                              int64_t work_bytes, void *stream);

/*
 * Right-padding collation of a ragged waveform buffer into a (B, T) float32 batch on the GPU: what lhotse's collate_audio
 * returns for mono cuts (DESIGN.md §3.1o).  Row b holds cut b's samples (int16 sources widened as q / 32768, exactly as
 * B200FEAT_I16 is widened for the feature kernels; float32 sources as they are), then zeros up to T.
 */
/* Device scratch b200feat_collate_audio needs for B cuts (0 when B is negative). */
int64_t b200feat_collate_audio_work_bytes(int32_t B);

/* `src_dev` (B200FEAT_F32 or B200FEAT_I16, `src_elems` elements; 16-byte aligned for F32, 8-byte for I16) holds cut b's
 * `lens[b]` samples from element `offsets[b]` (host arrays of B).  Checks the tables on the host before anything touches the
 * device (a negative offset or length, a length above T, samples outside the source buffer, an unknown dtype: each its own
 * message), copies them to `work_dev` and launches one kernel, asynchronously on `stream`.  Every element of the (B, T)
 * output `out_dev` is written exactly once, zeros included; elements outside it are not touched.  Errors are reported
 * through `h` (b200feat_last_error) when it is not NULL, and through b200feat_global_error. */
int b200feat_collate_audio(b200feat_handle *h, const void *src_dev, int32_t dt, int64_t src_elems, const int64_t *offsets,
                           const int64_t *lens, int32_t B, int64_t T, float *out_dev, void *work_dev, int64_t work_bytes,
                           void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B200FEAT_H_ */
