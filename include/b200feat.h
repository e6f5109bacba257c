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

#ifdef __cplusplus
}
#endif
#endif /* B200FEAT_H_ */
