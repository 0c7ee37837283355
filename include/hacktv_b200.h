/* hacktv_b200 - the C-ABI of the H100-native composite-video -> IQ hot path.
 *
 * This header is the drop-in boundary. Everything here is `extern "C"`, plain
 * pointers and sizes; no CUDA, torch or C++ types appear in any signature
 * (a CUDA stream is passed as an opaque `void *`).
 *
 * Each entry point replaces one piece of fsphil/hacktv's encoder interface.
 * "ref" = the reference's src/ directory; the adapter a hacktv maintainer adds
 * (video_b200.c, which implements video.h's vid_* symbols on top of these) is
 * shown in INTEGRATION.md and lives in integration/video_b200.c.
 *
 *   htv_config_t            <- vid_config_t               ref video.h:125-292 (hot-path subset, same names)
 *   htv_modes[], htv_find_mode <- vid_configs[]           ref video.c:1956-2008, hacktv.c:1078-1087
 *   htv_init                <- vid_init                   ref video.c:3812-4704
 *   htv_free                <- vid_free                   ref video.c:4706-4843
 *   htv_info                <- vid_info                   ref video.c:4846-4860
 *   htv_get_framebuffer_length <- vid_get_framebuffer_length  ref video.c:4862-4865
 *   htv_next_line           <- vid_next_line              ref video.c:4936-4952
 *   htv_line_t              <- vid_line_t                 ref video.h:306-329
 *   htv_av_t + callbacks    <- av_t, av_read_video_t ...  ref av.h:64-116, video.c:4873-4904, 3280
 *   htv_av_test_open        <- av_test_open               ref av_test.c:71-205
 *   htv_rf_t, htv_rf_write, htv_rf_close <- rf_t, rf_write, rf_close   ref rf.h:39-54, rf.c:23-51
 *   htv_rf_file_open        <- rf_file_open (int16 only)  ref rf_file.c:290-373
 *   htv_render / htv_render_host: NOT in the reference - the batched extension a
 *       per-line C call cannot replace (SURVEY.md §8b): N scan lines per call.
 *
 * Error convention follows the reference (video.h:45-47): 0 OK, -1 error,
 * -2 out of memory; htv_next_line returns NULL at end of stream.
 * Without a usable CUDA device htv_init fails with HTV_ERROR and a message on
 * stderr - there is no CPU fallback.
 */
#ifndef HACKTV_B200_H
#define HACKTV_B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HTV_OK             0
#define HTV_ERROR         -1
#define HTV_OUT_OF_MEMORY -2

/* output_type (ref rf.h:26-28) */
#define HTV_INT16_COMPLEX 0
#define HTV_INT16_REAL    1
/* sample type of the rendered stream, as the file sink's -t/--type (ref rf.h:31-36); htv_set_sample_type */
#define HTV_TYPE_UINT8  0
#define HTV_TYPE_INT8   1
#define HTV_TYPE_UINT16 2
#define HTV_TYPE_INT16  3
#define HTV_TYPE_INT32  4
#define HTV_TYPE_FLOAT  5
/* modulation (ref video.h:71-74) */
#define HTV_NONE 0
#define HTV_AM   1
#define HTV_VSB  2
#define HTV_FM   3
/* type (ref video.h:49-59); only these two rasters are on the hot path */
#define HTV_RASTER_625 0
#define HTV_RASTER_525 1
/* colour_mode (ref video.h:76-82) */
#define HTV_MONOCHROME 0
#define HTV_PAL        1
#define HTV_NTSC       2
#define HTV_SECAM      3
/* audio pre-emphasis (ref video.h:84-88) */
#define HTV_50US 1
#define HTV_75US 2
#define HTV_J17  3

/* The hot-path subset of vid_config_t, same field names and meaning. */
typedef struct {
	int32_t output_type;
	int32_t modulation;
	double video_bw;
	double vsb_upper_bw;
	double vsb_lower_bw;
	double level;
	int32_t swap_iq;
	int32_t invert_video;
	int64_t offset;
	double video_level;
	double fm_mono_level;
	double am_audio_level;
	double nicam_level;
	int32_t type;
	int32_t lines;
	int64_t frame_rate_num;
	int64_t frame_rate_den;
	int32_t hline;
	int32_t interlaced;
	int32_t active_lines;
	int32_t vfilter;
	double hsync_width;
	double vsync_short_width;
	double vsync_long_width;
	double sync_rise;
	double white_level;
	double black_level;
	double blanking_level;
	double sync_level;
	double active_width;
	double active_left;
	double gamma;
	double rw_co;
	double gw_co;
	double bw_co;
	int32_t colour_mode;
	int32_t volume;
	int64_t colour_carrier_num;
	int64_t colour_carrier_den;
	double colour_bw;
	double burst_width;
	double burst_left;
	double burst_level;
	double burst_rise;
	double ev_co;
	double eu_co;
	double fm_mono_carrier;
	double fm_mono_deviation;
	int32_t fm_mono_preemph;
	/* S-Video (ref video.h:229, --s-video hacktv.c:1136-1148): luma and sync on I, the colour subcarrier and its burst
	 * on Q instead of added to I; the stream is then complex (htv_is_complex). PAL, NTSC and SECAM colour with
	 * output_type HTV_INT16_REAL and no modulation only; not with a pixel rate other than the sample rate. It takes
	 * what was this struct's padding word, so that the layout (and orc_params_t's, which keeps the word as padding)
	 * does not change */
	int32_t s_video;
	double nicam_carrier;
	double nicam_beta;
	double am_mono_carrier;
	/* FM video, modulation == HTV_FM (ref video.h:141-143, -D/--deviation hacktv.c:1109-1113).
	 * fm_energy_dispersal must be 0: no mode in scope uses it */
	double fm_level;
	double fm_deviation;
	double fm_energy_dispersal;
} htv_config_t;

typedef struct {
	const char *id;
	const htv_config_t *conf;
	const char *desc;
} htv_mode_t;

extern const htv_mode_t htv_modes[];
extern const htv_config_t *htv_find_mode(const char *id);
extern size_t htv_config_size(void);

/* ---- AV source (pull model, as the reference's av_t) ------------------- */

typedef struct {
	int width;                    /* pixels per row */
	int height;                   /* rows */
	const uint32_t *framebuffer;  /* RGBx, row-major, tightly packed */
	uint64_t serial;              /* changes whenever the pixel data changes; a source
	                                 that returns the same image every frame (the test
	                                 pattern) keeps it constant so the upload is skipped */
} htv_frame_t;

typedef int (*htv_read_video_t)(void *ctx, htv_frame_t *frame);
typedef int (*htv_read_audio_t)(void *ctx, const int16_t **samples, size_t *npairs);
typedef int (*htv_av_close_t)(void *ctx);

typedef struct {
	int width;                    /* set by htv_init: active_width */
	int height;                   /* set by htv_init: active_lines */
	void *ctx;
	htv_read_video_t read_video;  /* once per frame, at line 1 (ref video.c:4873-4881) */
	htv_read_audio_t read_audio;  /* 32 kHz stereo int16, any block size (ref video.c:3280) */
	/* Buffers handed out by the callbacks are read by cudaMemcpyAsync on the encoder's upload
	 * stream. Pageable memory is staged before the callback's caller returns (reusable at once,
	 * as with the reference); page-locked memory (cudaHostAlloc) is read asynchronously - full
	 * PCIe rate, overlapped with the kernels and the copy back - and must stay unchanged until
	 * the render call that pulled it has completed on its stream. */
	htv_av_close_t close;
} htv_av_t;

/* ---- parity with the reference (what "drop-in" means numerically) --------
 * Against the reference's CPU path on the same picture and sound (tests/test_gpu_*.py, tests/golden/):
 *  - bit-exact wherever the path is integer-only: raster, sync pulses, PAL / NTSC chroma, SECAM chroma (its
 *    fp64 IIR and Q31 FM recurrence are run as the reference runs them), the VSB / low-pass video filter, VBI
 *    overlays, the --pixelrate resampler, the channel combiner, NICAM-728 end to end;
 *  - within +-1 LSB of int16 wherever an FM / AM sound carrier contributes: those are the reference's Q31
 *    phasor recurrences (a floor in every step), evaluated here in closed form of the sample index; > 97 % of
 *    the samples are still exact;
 *  - within +-2 LSB when --offset is combined with sound carriers: the offset mixer is one more such
 *    recurrence and multiplies the carriers' +-1 by its own; without sound carriers it is +-1;
 *  - FM video (pal-fm, ntsc-fm, secam-fm) without a sound carrier: +-1 LSB for ever. With one, the modulating
 *    signal inherits that carrier's +-1 LSB and an FM modulator integrates its input: the output is the same
 *    signal up to a slowly wandering common rotation (a random walk of ~15 - 40 LUT steps = 2 - 6 mrad per
 *    1 000 lines), instantaneous frequency identical at > 99.5 % of the samples;
 *  - long streams: the closed forms hold to +-1 LSB at 34 s (all device-side rings wrapped) EXCEPT where the
 *    reference's own recurrence stops behaving like its ideal carrier - an FM carrier at a small rational
 *    fraction of the sample rate (NTSC-M at 13.5 Msps: 4.5 MHz = fs / 3) makes its phasor revisit the same few
 *    states, the floors stop averaging out and the REFERENCE runs slow by ~1e-5 Hz (0.35 LSB / s of sound
 *    carrier; tools/nco_drift.c). The same mode at 16 Msps does not show it. */

/* ---- encoder ----------------------------------------------------------- */

typedef struct htv_t htv_t;

typedef struct {
	int16_t *output;   /* int16 I,Q interleaved, 2 * width values (Q = 0 for real modes) */
	int width;
	int frame;         /* 1-based */
	int line;          /* 1-based */
} htv_line_t;

extern int htv_init(htv_t **s, unsigned int sample_rate, unsigned int pixel_rate, const htv_config_t *conf);
/* Device placement (SURVEY.md section 8e: one RF channel per GPU, channel c -> device c mod N). htv_init
 * binds the encoder to the calling thread's current CUDA device; htv_init_on to CUDA device `device`
 * (0 .. htv_device_count() - 1; -1 = current). Every later call on the encoder runs on that device
 * whatever the calling thread's current device is, and leaves the caller's current device unchanged: a
 * C host drives N encoders on N GPUs from one process, from one thread or one thread per encoder (an
 * encoder itself is not re-entrant: one call at a time per htv_t). Device pointers handed to
 * htv_render / htv_render_add must belong to the encoder's device (or be peer-accessible from it). */
extern int htv_init_on(htv_t **s, int device, unsigned int sample_rate, unsigned int pixel_rate, const htv_config_t *conf);
extern int htv_device_count(void);
extern int htv_device(const htv_t *s);
extern void htv_free(htv_t *s);
extern void htv_info(htv_t *s);
extern size_t htv_get_framebuffer_length(htv_t *s);
extern htv_av_t *htv_av(htv_t *s);
extern int htv_av_test_open(htv_av_t *av);
extern void htv_av_close(htv_av_t *av);
/* In-memory source: caller-owned RGBx pictures (av->width x av->height each, one per video frame,
 * cyclic) and 32 kHz stereo PCM (cyclic, `audio_block` pairs per read; 0 = all). `static_video`
 * != 0 promises the pictures never change, so each is uploaded once. Pointers are borrowed. */
extern int htv_av_memory_open(htv_av_t *av, const uint32_t *frames, size_t nframes,
	const int16_t *audio, size_t audio_pairs, size_t audio_block, int static_video);

/* VBI overlays - the hook the reference's VBI stages (teletext, WSS, VITS, VITC, CC608; registered
 * behind the raster and SECAM stages, ref video.c:4213-4357) need from the encoder: each of them adds an
 * int16 waveform to a finished line (vbidata_render, ref vbidata.c:186-239; wss_render first sets part of
 * line 23 to black, ref wss.c:182-185). The packet / waveform builders stay host code; once per frame, when
 * its first line is rendered, `read` reports the lines they touch: I[replace_from, replace_to) =
 * replace_value (skipped when from >= to), then I[x] += add[x] for the W samples of the line (int16 wrap;
 * NULL = nothing to add). At most one entry per line; entries must leave the first 40 samples of a line
 * alone (VBI data does: that is sync and back porch). The arrays need only stay valid until `read` returns. */
typedef struct {
	int line;                     /* 1-based, as the reference counts */
	int replace_from, replace_to;
	int replace_value;
	const int16_t *add;
} htv_vbi_line_t;
typedef int (*htv_read_vbi_t)(void *ctx, int frame /* 1-based */, const htv_vbi_line_t **lines, int *nlines);
extern int htv_set_vbi_source(htv_t *s, htv_read_vbi_t read, void *ctx);

extern htv_line_t *htv_next_line(htv_t *s);
/* htv_next_line hands out lines of a frame held in pinned host memory. With prefetch on, the following frame
 * is rendered and copied while the caller consumes the current one (two pinned frames), so a
 * vid_next_line + rf_write loop is bounded by the consumer, not by a GPU round trip per frame. The price:
 * the AV source is pulled one frame earlier than the reference would pull it - fine for sources that do not
 * end (test pattern, live capture), wrong by one frame at the end of a file. Off by default. */
extern int htv_set_prefetch(htv_t *s, int on);

/* Batched extension. Renders the next `nlines` scan lines of the stream.
 * htv_render: `d_out` is DEVICE memory (at least htv_samples_per_line(s) *
 *   nlines * htv_bytes_per_sample(s) bytes); work is enqueued on `cuda_stream`
 *   (a cudaStream_t, or NULL for the default stream) and the call returns
 *   without synchronising.
 * htv_render_host: `h_out` is HOST memory; the call uploads what the batch
 *   needs, renders, copies the result back and returns when it is there.
 * Both return HTV_OK or an error; *nsamples (may be NULL) receives the number
 * of samples produced. `d_out` must be aligned to the widest access the encoder's store (and
 * htv_render_add's loads) make: 16 bytes where the split and FM-video modulators store four
 * complex int16 samples at once (4 divides the line width), 8 for four real ones, otherwise one
 * sample (htv_bytes_per_sample). A pointer a whole number of lines into a 16-byte aligned buffer
 * always qualifies - the reference's two-channel alignment, one line in, at any width. A
 * misaligned pointer is refused with HTV_ERROR. Output layout is what the reference's file sink writes
 * (rf_file.c:97-116, 226-233): int16 I,Q interleaved for complex modes, int16
 * I only for real modes. With htv_set_sample_type the buffer holds that type
 * instead (the pointer keeps its int16_t type; size it in bytes). */
extern int htv_render(htv_t *s, int nlines, int16_t *d_out, size_t *nsamples, void *cuda_stream);
extern int htv_render_host(htv_t *s, int nlines, int16_t *h_out, size_t *nsamples);

/* Sample type of what htv_render / htv_render_host write: HTV_TYPE_UINT8 .. HTV_TYPE_FLOAT, each value converted
 * from the int16 the encoder computes exactly as the reference's file sink converts it (ref rf_file.c, -t/--type):
 * uint8 (x + 32768) >> 8, int8 x >> 8, uint16 x + 32768, int32 x * 65537, float x / 32767 (rounded from a double
 * product). The conversion is the last step of the store, after --offset and the channel combiner (htv_set_passthru
 * still adds in int16). Default HTV_TYPE_INT16. Allowed only before the first line is rendered; an unknown type is
 * refused. htv_bytes_per_sample follows it. htv_render_add (an int16 sum) and htv_next_line (int16 lines, as
 * vid_next_line) refuse any other type. */
extern int htv_set_sample_type(htv_t *s, int type);
extern int htv_sample_type(const htv_t *s);
/* d_dst[i] = the `type` form of d_src[i] over nvalues int16 values in device memory (I and Q alike), stream-ordered
 * on cuda_stream. Both pointers 16-byte aligned. For streams that already exist: a wideband sum built with
 * htv_render_add, converted once at the end. */
extern int htv_convert(void *d_dst, int type, const int16_t *d_src, size_t nvalues, void *cuda_stream);

/* Channel combiner - replaces the reference's `--passthru` stage (vid_config_t.passthru
 * video.h:158; _vid_passthru_process video.c:3517-3541, set-up 4607-4634): an external int16
 * stream is added to this encoder's output, component by component with int16 wrap, as the
 * very last step (after --offset). Three forms:
 *  htv_set_passthru: an fread-like source of int16 complex samples (I,Q interleaved, as the
 *    reference reads them); `read` returns the complex samples delivered, a short count means
 *    end of stream (only whole lines are added after that, as in the reference). Must be
 *    installed before the first line is rendered. As in the reference the first
 *    htv_passthru_delay_lines() lines of the external stream are consumed without being
 *    used (they meet the pipeline's fill lines): output line j gets external line j + delay.
 *  htv_render_add: like htv_render, but adds this encoder's lines INTO what `d_out` already
 *    holds (same layout) - k channels with different --offset rendered into one wideband
 *    buffer without the stream ever leaving HBM. The caller picks the alignment.
 *  htv_mix_add: d_acc[i] += d_in[i] (int16 wrap) over nvalues int16 values, both device
 *    (or peer-mapped) pointers, 16-byte aligned; for streams that already exist. */
typedef size_t (*htv_passthru_read_t)(void *ctx, int16_t *iq, size_t ncomplex);
extern int htv_set_passthru(htv_t *s, htv_passthru_read_t read, void *ctx);
extern int htv_passthru_delay_lines(const htv_t *s);
extern int htv_render_add(htv_t *s, int nlines, int16_t *d_out, size_t *nsamples, void *cuda_stream);
extern int htv_mix_add(int16_t *d_acc, const int16_t *d_in, size_t nvalues, void *cuda_stream);

/* Geometry / state accessors (fields hacktv.c reads from vid_t, ref video.h:358-420) */
extern int htv_samples_per_line(const htv_t *s);   /* vid_t.width */
extern int htv_half_line(const htv_t *s);          /* vid_t.half_width */
extern void htv_signal_levels(const htv_t *s, int levels[4]);   /* vid_t.white_level, black_level, blanking_level, sync_level */
extern int htv_active_width(const htv_t *s);
extern int htv_active_lines(const htv_t *s);
extern int htv_lines_per_frame(const htv_t *s);
extern int htv_sample_rate(const htv_t *s);
extern int htv_is_complex(const htv_t *s);
extern int htv_bytes_per_sample(const htv_t *s);   /* int16: 4 complex, 2 real; other sample types their size */
extern int64_t htv_lines_rendered(const htv_t *s);
/* Kernel launches issued by this encoder since htv_init (for bench accounting) */
extern uint64_t htv_kernel_launches(const htv_t *s);
/* The line kernel(s) the most recent render launched, with their template arguments, e.g.
 * "k_line<VF=1,HQ=1,FULL=0,CSAT=1,MAXT=384,SRC=0,SND=-1,WC=0>", or for SECAM
 * "k_sec_raster<FULL=1,MAXT=384> + k_line<...,SRC=1,...>"; "" before the first render. A store that converts to
 * another sample type than int16 appends it: ",ST=int8" compiled in, ",ST=-1:float" chosen at run time (k_line), or
 * " ST=-1:float" after the split, FM-video and --pixelrate modulators. Read-only diagnostic:
 * the string belongs to the encoder and changes with the next render. */
extern const char *htv_line_kernel(const htv_t *s);
/* What the SECAM chrominance chain did since htv_init (DESIGN §6), summed over its launches; all zero for other
 * colour modes. A launch is one sub-batch of a render call; a pass is one round of k_sec_refine + the list kernels; the
 * work list holds the lines whose FM recurrence is re-run in full, by k_sec_fm_list (one warp per line) or, for a list
 * longer than 2048 lines, by k_sec_fm_list_t (one thread per line). Filled from counts the chain copies to the host
 * anyway: reading it costs no device work. */
typedef struct {
	int64_t launches;                     /* chain launches */
	int64_t passes;                       /* refinement passes */
	int64_t final_odd, final_even;        /* launches whose last pass had an odd / even number */
	int64_t recomputed;                   /* lines k_sec_refine recomputed */
	int64_t listed_warp, listed_thread;   /* listed lines finished by k_sec_fm_list / k_sec_fm_list_t */
	int64_t repredict_odd, repredict_even;/* second proposals of k_sec_predict after an odd / even pass */
	int32_t passes_max;                   /* most passes one launch needed */
	int32_t list_max;                     /* longest work list of one pass */
} htv_secam_chain_t;
extern int htv_secam_chain(const htv_t *s, htv_secam_chain_t *out);
/* Duration of the dominant kernel's (k_mod) most recent launch, measured with CUDA
 * events on the stream it ran on (0 if timing is off), and the scan lines that launch covered. */
extern void htv_set_kernel_timing(htv_t *s, int on);
extern float htv_last_line_kernel_ms(htv_t *s);
extern int htv_last_line_kernel_lines(const htv_t *s);

/* ---- host-only table generation (no GPU needed; used by htv_init) ------ */

typedef struct htv_tables_t htv_tables_t;

extern htv_tables_t *htv_tables_create(const htv_config_t *conf, unsigned int sample_rate);
/* The sample-rate side of vid_init(sample_rate, pixel_rate != sample_rate): everything from the
 * --pixelrate resampler on (ref _init_vresampler video.c:3627-3651, 4361-4368; fir_int16_resampler_init
 * fir.c:393-428): the polyphase taps ("rs_taps", "rs_geometry" = I, D, taps per phase, raster width), the
 * video filter and sound carriers at sample_rate, and the extra line of pipeline lead. NULL for rate
 * pairs whose line width would vary and for FM video. pixel_rate 0 or == sample_rate: htv_tables_create. */
extern htv_tables_t *htv_tables_create2(const htv_config_t *conf, unsigned int sample_rate, unsigned int pixel_rate);
extern void htv_tables_free(htv_tables_t *t);
/* Named int32 views for tests: "sync0".."sync4", "sync_off", "burst_win",
 * "chroma_taps", "vsb_itaps", "vsb_qtaps", "levels", "nicam_taps", "geometry",
 * "secam_lpf", "secam_notch", "rs_taps", "rs_geometry". Returns NULL for an unknown / absent table. */
extern const int32_t *htv_tables_get(htv_tables_t *t, const char *name, int *count);

/* ---- RF sink (int16 file sink only) ------------------------------------ */

typedef int (*htv_rf_write_t)(void *ctx, const int16_t *iq_data, size_t samples);
typedef int (*htv_rf_close_t)(void *ctx);

typedef struct {
	void *ctx;
	htv_rf_write_t write;
	htv_rf_close_t close;
} htv_rf_t;

extern int htv_rf_write(htv_rf_t *s, const int16_t *iq_data, size_t samples);
extern int htv_rf_close(htv_rf_t *s);
extern int htv_rf_file_open(htv_rf_t *s, const char *filename, int complex);

/* The built-in test source's data, exposed for tests (ref av_test.c:94-196) */
extern void htv_test_pattern(int width, int height, uint32_t *rgb);
extern size_t htv_test_tone_pairs(void);
extern void htv_test_tone(int16_t *pcm);

extern const char *htv_version(void);

#ifdef __cplusplus
}
#endif

#endif
