/* hacktv_b200 - C host layer: the encoder object behind the C-ABI.
 *
 * Mirrors the reference's vid_t life cycle (ref video.c:3812-4952, hacktv.c:1440-1601):
 * init -> caller installs an AV source -> pull lines -> free. The per-line pthread
 * pipeline of the reference is replaced by batched device launches: a call renders N
 * scan lines; htv_next_line() is a view over a pinned host buffer refilled one frame
 * at a time.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "htv_internal.h"
#include "htv_sample_type.h"

/* Picture slots on the device and new pictures per launch sequence: with 16 slots and at most 7
 * new pictures (+ 1 carried over) per chunk, the uploads of chunk c touch no slot chunk c-1 reads,
 * so they may run (on the upload stream) while chunk c-1 is still computing. */
#define MAX_FRAME_SLOTS 16
#define MAX_NEW_FRAMES 7
#define MAX_CHUNK_SECONDS 4.0
_Static_assert(MAX_NEW_FRAMES <= HTV_INGEST_MAX, "a call's new pictures are one k_ingest list at most");
#define PT_MAX_LINES 4096

struct htv_t {
	htv_tables_t *tab;
	htv_dev_t *dev;
	htv_av_t av;

	int W, lines, complex, bps;
	int type;                     /* HTV_TYPE_* of the rendered stream (htv_set_sample_type); bps follows it */

	/* stream position */
	/* --pixelrate (ref vid_init video.c:3839, _init_vresampler 3627-3651): the raster side - tables, pictures,
	 * frame map, VBI overlays - lives in a second device context built at the pixel rate; the resampler,
	 * video filter, sound carriers and output stay in `dev` at the sample rate. Without a resampler
	 * rtab == tab and rdev == dev. */
	struct htv_tables_t *rtab;
	htv_dev_t *rdev;
	int64_t next_line;            /* next scan line to render (0 = frame 1 line 1) */

	/* video frames */
	int64_t cur_frame;            /* 0-based index of the last frame pulled, -1 none */
	int cur_slot;                 /* its slot, -1 = no picture (black) */
	int prev_slot;                /* the slot of frame cur_frame - 1 */
	uint64_t cur_serial;
	int have_serial;
	int next_slot;
	htv_read_video_device_t dev_read;   /* htv_set_video_device_source: used while av.read_video is NULL */
	void *dev_ctx;

	/* audio */
	int64_t audio_have;           /* source pairs uploaded so far (absolute count) */
	htv_device_audio_t pend;      /* rest of a source block larger than one ring piece: sent before the next read */
	int pend_dev;                 /* ... and whether it is in device memory */
	htv_read_audio_device_t adev_read;  /* htv_set_audio_device_source: used while av.read_audio is NULL */
	void *adev_ctx;
	int16_t *zeros;

	/* VBI overlays pulled from the source, kept until their line has been rendered */
	htv_read_vbi_t vbi_read;
	void *vbi_ctx;
	struct { long long line; int from, to, value; int16_t *add; } *ov;
	int nov, ov_cap;

	/* channel combiner (ref --passthru, video.c:3517-3541, 4607-4634) */
	htv_passthru_read_t pt_read;
	void *pt_ctx;
	int pt_started;
	int16_t *pt_host;             /* pinned staging, PT_MAX_LINES lines in output layout */
	int16_t *pt_dev;
	int16_t *pt_tmp;              /* complex scratch for real-output modes */

	/* htv_render_host: two device staging buffers, rendering of one piece overlaps the
	 * device-to-host copy of the previous one */
	int16_t *d_stage[2];
	size_t d_stage_bytes;
	void *st_compute, *st_copy;
	void *ev_rendered[2], *ev_copied[2];

	unsigned piece_i;             /* pieces queued so far (staging buffer = piece_i & 1) */

	/* htv_next_line view: two pinned frames - while the caller walks one, the next is rendered and copied */
	int16_t *h_frame[2];          /* pinned, one frame of output each */
	int h_cur;                    /* the frame being handed out */
	int h_lines;                  /* lines held */
	int h_pos;                    /* next line to hand out */
	int64_t h_first_line;
	int prefetch;                 /* htv_set_prefetch */
	int pf_pending, pf_lines;     /* a frame is in flight into h_frame[h_cur ^ 1] */
	int64_t pf_first_line;
	void *ev_frame[2];
	int16_t *h_iq;                /* interleaved scratch for real modes */
	htv_line_t line;
};

static void drop_overlays_before(htv_t *s, long long line);

const char *htv_version(void) { return("hacktv_b200 0.1 (sm_90a)"); }

const htv_config_t *htv_find_mode(const char *id)
{
	const htv_mode_t *m;
	if(!id) return(NULL);
	for(m = htv_modes; m->id; m++) if(strcmp(m->id, id) == 0) return(m->conf);
	return(NULL);
}

size_t htv_config_size(void) { return(sizeof(htv_config_t)); }

int htv_init(htv_t **out, unsigned int sample_rate, unsigned int pixel_rate, const htv_config_t *conf)
{
	return(htv_init_on(out, -1, sample_rate, pixel_rate, conf));
}

int htv_device_count(void) { return(htv_dev_count()); }
int htv_device(const htv_t *s) { return(s ? htv_dev_device(s->dev) : -1); }

int htv_init_on(htv_t **out, int device, unsigned int sample_rate, unsigned int pixel_rate, const htv_config_t *conf)
{
	htv_t *s;
	char err[256];

	if(!out) return(HTV_ERROR);
	*out = NULL;
	s = calloc(1, sizeof(htv_t));
	if(!s) return(HTV_OUT_OF_MEMORY);

	s->tab = htv_tables_create2(conf, sample_rate, pixel_rate);
	if(!s->tab) { free(s); return(HTV_ERROR); }
	s->rtab = s->tab;
	if(s->tab->rs_taps)
	{
		/* the raster side at the pixel rate: same mode, no sound carriers, filter or mixers */
		htv_config_t rc = *conf;
		rc.vfilter = 0; rc.offset = 0; rc.swap_iq = 0;
		rc.fm_mono_level = 0; rc.nicam_level = 0; rc.am_audio_level = 0;
		s->rtab = htv_tables_create(&rc, pixel_rate);
		if(!s->rtab || s->rtab->dp.W != s->tab->rs_wp)
		{
			htv_tables_free(s->rtab != s->tab ? s->rtab : NULL);
			htv_tables_free(s->tab);
			free(s);
			return(HTV_ERROR);
		}
		s->rtab->raster_only = 1;
		/* the raster context's kernels are planned first, so that a pixel-rate line they cannot hold is refused
		 * before anything is allocated or launched on the device */
		if(htv_dev_plan_name(s->rtab, s->rtab->dp.sample_type, err, sizeof(err)) != HTV_OK)
		{
			fprintf(stderr, "hacktv_b200: cannot initialise the CUDA encoder: %s\n", err);
			htv_tables_free(s->rtab);
			htv_tables_free(s->tab);
			free(s);
			return(HTV_ERROR);
		}
	}

	/* No GPU, no encoder: there is deliberately no CPU fallback */
	s->dev = htv_dev_create(s->tab, MAX_FRAME_SLOTS, device, err, sizeof(err));
	s->rdev = s->dev;
	if(s->dev && s->rtab != s->tab)
	{
		s->rdev = htv_dev_create(s->rtab, MAX_FRAME_SLOTS, htv_dev_device(s->dev), err, sizeof(err));
		if(!s->rdev) { htv_dev_destroy(s->dev); s->dev = NULL; }
	}
	if(!s->dev)
	{
		fprintf(stderr, "hacktv_b200: cannot initialise the CUDA encoder: %s\n", err);
		if(s->rtab != s->tab) htv_tables_free(s->rtab);
		htv_tables_free(s->tab);
		free(s);
		return(HTV_ERROR);
	}

	s->W = s->tab->dp.W;
	s->lines = s->tab->dp.lines;
	s->complex = s->tab->dp.complex_out;
	s->type = HTV_TYPE_INT16;
	s->bps = htv_st_bytes(s->type, s->complex);
	s->cur_frame = -1;
	s->cur_slot = -1;
	s->prev_slot = -1;
	s->av.width = s->rtab->dp.active_width;
	s->av.height = s->rtab->dp.active_lines;
	s->zeros = htv_dev_alloc_pinned(65536 * 2 * sizeof(int16_t));    /* pinned: uploads stay asynchronous */
	if(!s->zeros) { htv_free(s); return(HTV_OUT_OF_MEMORY); }
	memset(s->zeros, 0, 65536 * 2 * sizeof(int16_t));
	*out = s;
	return(HTV_OK);
}

void htv_av_close(htv_av_t *av)
{
	if(av && av->close) av->close(av->ctx);
	if(av) { av->ctx = NULL; av->read_video = NULL; av->read_audio = NULL; av->close = NULL; }
}

void htv_free(htv_t *s)
{
	if(!s) return;
	htv_av_close(&s->av);
	if(s->dev)
	{
		htv_dev_free(s->dev, s->d_stage[0]);
		htv_dev_free(s->dev, s->d_stage[1]);
		htv_dev_free(s->dev, s->pt_dev);
		htv_dev_event_free(s->ev_rendered[0]); htv_dev_event_free(s->ev_rendered[1]);
		htv_dev_event_free(s->ev_copied[0]); htv_dev_event_free(s->ev_copied[1]);
		htv_dev_stream_free(s->st_compute); htv_dev_stream_free(s->st_copy);
		if(s->rdev && s->rdev != s->dev) htv_dev_destroy(s->rdev);
		htv_dev_destroy(s->dev);
	}
	drop_overlays_before(s, 0x7FFFFFFFFFFFFFFFLL);
	free(s->ov);
	htv_dev_free_pinned(s->h_frame[0]);
	htv_dev_free_pinned(s->h_frame[1]);
	htv_dev_free_pinned(s->pt_host);
	free(s->pt_tmp);
	free(s->h_iq);
	htv_dev_free_pinned(s->zeros);
	if(s->rtab != s->tab) htv_tables_free(s->rtab);
	htv_tables_free(s->tab);
	free(s);
}

void htv_info(htv_t *s)
{
	const htv_config_t *c = &s->tab->conf;
	fprintf(stderr, "Video: %dx%d %.2f fps (full frame %dx%d)\n",
		s->rtab->dp.active_width, c->active_lines,
		(double) c->frame_rate_num / c->frame_rate_den, s->rtab->dp.W, c->lines);
	if(s->rtab != s->tab) fprintf(stderr, "Pixel rate: %d\n", (int) s->rtab->rate);
	fprintf(stderr, "Sample rate: %d\n", (int) s->tab->rate);
}

size_t htv_get_framebuffer_length(htv_t *s)
{
	return(sizeof(uint32_t) * s->rtab->dp.active_width * s->tab->conf.active_lines);
}

htv_av_t *htv_av(htv_t *s) { return(&s->av); }
int htv_samples_per_line(const htv_t *s) { return(s->W); }
int htv_half_line(const htv_t *s) { return(s->rtab->dp.half_width); }   /* of the raster (VBI stages draw there) */
void htv_signal_levels(const htv_t *s, int levels[4]) { htv_tables_levels(s->tab, levels); }
int htv_active_width(const htv_t *s) { return(s->rtab->dp.active_width); }
int htv_active_lines(const htv_t *s) { return(s->tab->dp.active_lines); }
int htv_lines_per_frame(const htv_t *s) { return(s->lines); }
int htv_sample_rate(const htv_t *s) { return((int) s->tab->rate); }
int htv_is_complex(const htv_t *s) { return(s->complex); }
int htv_bytes_per_sample(const htv_t *s) { return(s->bps); }
int htv_sample_type(const htv_t *s) { return(s ? s->type : -1); }

int htv_set_sample_type(htv_t *s, int type)
{
	if(!s) return(HTV_ERROR);
	if(!htv_st_size(type))
	{
		fprintf(stderr, "hacktv_b200: unknown sample type %d (HTV_TYPE_UINT8 .. HTV_TYPE_FLOAT)\n", type);
		return(HTV_ERROR);
	}
	if(s->next_line != 0)
	{
		fprintf(stderr, "hacktv_b200: the sample type must be set before the first line is rendered\n");
		return(HTV_ERROR);
	}
	/* the output context (with --pixelrate the raster side stays int16) */
	if(htv_dev_set_sample_type(s->dev, type) != HTV_OK) return(HTV_ERROR);
	s->type = type;
	s->bps = htv_st_bytes(type, s->complex);
	return(HTV_OK);
}

int htv_convert(void *d_dst, int type, const int16_t *d_src, size_t nvalues, void *cuda_stream)
{
	if(!htv_st_size(type))
	{
		fprintf(stderr, "hacktv_b200: unknown sample type %d (HTV_TYPE_UINT8 .. HTV_TYPE_FLOAT)\n", type);
		return(HTV_ERROR);
	}
	if(nvalues && (!d_dst || !d_src || ((uintptr_t) d_dst & 15) || ((uintptr_t) d_src & 15)))
	{
		fprintf(stderr, "hacktv_b200: htv_convert needs 16-byte aligned device pointers\n");
		return(HTV_ERROR);
	}
	return(htv_dev_convert(d_dst, type, d_src, nvalues, cuda_stream));
}
int64_t htv_lines_rendered(const htv_t *s) { return(s->next_line); }
uint64_t htv_kernel_launches(const htv_t *s) { return(htv_dev_launches(s->dev)); }
const char *htv_line_kernel(const htv_t *s) { return(htv_dev_line_kernel(s->dev)); }
int htv_secam_chain(const htv_t *s, htv_secam_chain_t *out)
{
	if(!s || !out) return(HTV_ERROR);
	htv_dev_secam_chain(s->dev, out);
	return(HTV_OK);
}
void htv_set_kernel_timing(htv_t *s, int on) { htv_dev_set_timing(s->dev, on); }
float htv_last_line_kernel_ms(htv_t *s) { return(htv_dev_last_line_ms(s->dev)); }
int htv_last_line_kernel_lines(const htv_t *s) { return(htv_dev_last_line_count(s->dev)); }

int htv_set_video_device_source(htv_t *s, htv_read_video_device_t read, void *ctx)
{
	if(!s) return(HTV_ERROR);
	if(s->next_line != 0)
	{
		fprintf(stderr, "hacktv_b200: the video source must be set before the first line is rendered\n");
		return(HTV_ERROR);
	}
	s->av.read_video = NULL;
	s->dev_read = read;
	s->dev_ctx = ctx;
	return(HTV_OK);
}

int htv_set_audio_device_source(htv_t *s, htv_read_audio_device_t read, void *ctx)
{
	if(!s) return(HTV_ERROR);
	if(s->next_line != 0)
	{
		fprintf(stderr, "hacktv_b200: the sound source must be set before the first line is rendered\n");
		return(HTV_ERROR);
	}
	s->av.read_audio = NULL;
	s->adev_read = read;
	s->adev_ctx = ctx;
	return(HTV_OK);
}

/* audio fetches completed up to and including audio-clock sample m (ref video.c:3273-3276) */
static int64_t fetches_by(int64_t m, unsigned int rate)
{
	return((int64_t) (((unsigned long long) (m + 1) * HTV_AUDIO_RATE) / rate));
}

/* host PCM (read_audio's interleaved int16 pairs) described as a block */
static htv_device_audio_t host_block(const int16_t *pcm, size_t npairs)
{
	htv_device_audio_t b;
	b.data = pcm; b.npairs = npairs; b.format = HTV_PCM_INT16;
	b.stride_pair = 2 * sizeof(int16_t); b.stride_ch = sizeof(int16_t);
	return(b);
}

/* Make source audio available on the device up to pair index `need` (exclusive). A source may hand
 * over blocks of any size (ref video.c:3280): one larger than a quarter of the device ring goes up in
 * ring-sized pieces, the remainder kept for the next calls - nothing is dropped. Host blocks are copied
 * up, device blocks (htv_set_audio_device_source) converted into the ring on the device. */
static int pull_audio(htv_t *s, int64_t need, void *stream)
{
	const size_t piece = htv_dev_audio_ring_pairs() / 4;
	while(s->audio_have < need)
	{
		htv_device_audio_t b = s->pend;
		int dev = s->pend_dev, r;

		if(!b.npairs)
		{
			memset(&b, 0, sizeof(b));
			dev = 0;
			if(s->av.read_audio)
			{
				const int16_t *pcm = NULL;
				size_t n = 0;
				s->adev_read = NULL;                     /* a read_audio installed after a device source replaces it */
				if(s->av.read_audio(s->av.ctx, &pcm, &n) != HTV_OK) { s->av.read_audio = NULL; pcm = NULL; n = 0; }
				b = host_block(pcm, n);
			}
			else if(s->adev_read)
			{
				/* a device source ends at its first empty block */
				if(s->adev_read(s->adev_ctx, &b) == HTV_OK && b.data && b.npairs) dev = 1;
				else { s->adev_read = NULL; b.data = NULL; }
			}
			if(!b.data || b.npairs == 0)
			{
				/* no audio from the source: silence (ref video.c:3298-3303) */
				size_t n = (size_t) (need - s->audio_have);
				b = host_block(s->zeros, n > 65536 ? 65536 : n);
			}
		}
		s->pend.npairs = 0;
		if(b.npairs > piece)
		{
			/* only what this render call needs now (at most a piece): the device ring holds about 32 s */
			size_t take = (size_t) (need - s->audio_have);
			if(take > piece) take = piece;
			if(take < b.npairs)
			{
				s->pend = b;
				s->pend.data = (const char *) b.data + (int64_t) take * b.stride_pair;
				s->pend.npairs = b.npairs - take;
				s->pend_dev = dev;
				b.npairs = take;
			}
		}
		r = dev ? htv_dev_ingest_audio(s->dev, s->audio_have, &b, stream)
			: htv_dev_upload_audio(s->dev, s->audio_have, (const int16_t *) b.data, b.npairs, stream);
		if(r != HTV_OK) return(r);
		s->audio_have += (int64_t) b.npairs;
	}
	return(HTV_OK);
}

/* ---- channel combiner -----------------------------------------------------
 * The reference adds an external int16 complex stream to its own output, line by line, as
 * the last stage before the sink (ref _vid_passthru_process video.c:3517-3541). Because that
 * stage also runs on the pipeline's fill lines, the first `delay` lines of the external
 * stream are consumed and dropped with them: output line j receives external line j + delay,
 * where delay = 1 with a video filter and 0 without (measured on the reference, see
 * tests/test_oracle_vs_ref.py::test_passthru_alignment). A stream that ends adds whole lines
 * only (the `fread() == 0 -> return` at video.c:3530). */
int htv_passthru_delay_lines(const htv_t *s) { return(s->tab->dp.shift / s->tab->dp.W); }   /* 0, 1; 2 with a resampler and a filter */

int htv_set_passthru(htv_t *s, htv_passthru_read_t read, void *ctx)
{
	if(!s) return(HTV_ERROR);
	if(s->next_line != 0 && read) return(HTV_ERROR);      /* as in the reference: fixed at init */
	s->pt_read = read;
	s->pt_ctx = ctx;
	s->pt_started = 0;
	return(HTV_OK);
}

/* Stage the next n lines of the external stream on the device; returns whole lines available */
static int pull_passthru(htv_t *s, int n, void *stream)
{
	const size_t W = (size_t) s->W;
	size_t got;
	int lines, r;

	if(!s->pt_host)
	{
		s->pt_host = htv_dev_alloc_pinned(sizeof(int16_t) * 2 * W * PT_MAX_LINES);
		s->pt_dev = htv_dev_alloc(s->dev, sizeof(int16_t) * 2 * W * PT_MAX_LINES);
		if(!s->complex) s->pt_tmp = malloc(sizeof(int16_t) * 2 * W * PT_MAX_LINES);
		if(!s->pt_host || !s->pt_dev || (!s->complex && !s->pt_tmp)) return(-1);
	}
	/* the staging buffer may still be in flight from the previous chunk */
	if(htv_dev_sync(s->dev, stream) != HTV_OK) return(-1);
	if(!s->pt_started)
	{
		size_t skip = (size_t) htv_passthru_delay_lines(s) * W;
		s->pt_started = 1;
		if(skip && s->pt_read(s->pt_ctx, s->pt_host, skip) < skip) { s->pt_read = NULL; return(0); }
	}
	if(s->complex) got = s->pt_read(s->pt_ctx, s->pt_host, (size_t) n * W);
	else
	{
		/* real output carries I only (the file sink drops Q, ref rf_file.c:97-116) */
		size_t i;
		got = s->pt_read(s->pt_ctx, s->pt_tmp, (size_t) n * W);
		for(i = 0; i < got; i++) s->pt_host[i] = s->pt_tmp[i * 2];
	}
	if(got < (size_t) n * W) s->pt_read = NULL;           /* end of the external stream */
	lines = (int) (got / W);
	if(lines > 0)
	{
		/* int16 in the output layout whatever the sample type: the combiner adds before the conversion */
		r = htv_dev_memcpy_h2d(s->dev, s->pt_dev, s->pt_host, (size_t) lines * W * htv_st_bytes(HTV_TYPE_INT16, s->complex), stream);
		if(r != HTV_OK) return(-1);
	}
	return(lines);
}

/* ---- VBI overlays ------------------------------------------------------------
 * The reference's VBI stages (teletext, WSS, VITS, VITC, CC608: ref video.c:4213-4357) each add a
 * sparse int16 waveform to a finished raster line (vbidata_render, vbidata.c:186-239; WSS first sets
 * part of line 23 to black, wss.c:182-185). They stay host code: whoever builds the packets hands
 * the encoder, once per frame, the lines they touch; the raster kernel applies them. */
int htv_set_vbi_source(htv_t *s, htv_read_vbi_t read, void *ctx)
{
	if(!s) return(HTV_ERROR);
	s->vbi_read = read;
	s->vbi_ctx = ctx;
	return(HTV_OK);
}

static void drop_overlays_before(htv_t *s, long long line)
{
	int i, k = 0;
	for(i = 0; i < s->nov; i++)
	{
		if(s->ov[i].line < line) { free(s->ov[i].add); continue; }
		s->ov[k++] = s->ov[i];
	}
	s->nov = k;
}

#define MAX_VBI_LINES_PER_FRAME 64

/* Pull frame f's overlays (f 0-based), after its picture - as the reference's VBI stages run after the
 * frame was loaded (ref video.c:4873-4904, then the line processes) */
static void pull_overlays(htv_t *s, int64_t f)
{
	const htv_vbi_line_t *lines = NULL;
	int n = 0, i, j;
	if(s->vbi_read(s->vbi_ctx, (int) (f + 1), &lines, &n) != HTV_OK || n <= 0 || !lines) return;
	if(n > MAX_VBI_LINES_PER_FRAME) n = MAX_VBI_LINES_PER_FRAME;
	if(s->nov + n > s->ov_cap)
	{
		s->ov_cap = (s->nov + n) * 2;
		s->ov = realloc(s->ov, sizeof(*s->ov) * s->ov_cap);
	}
	for(i = 0; i < n; i++)
	{
		const long long gl = (long long) f * s->lines + (lines[i].line - 1);
		if(lines[i].line < 1 || lines[i].line > s->lines) continue;
		/* keep the table sorted by line (frames arrive in order; lines of a frame may not) */
		for(j = s->nov; j > 0 && s->ov[j - 1].line > gl; j--) s->ov[j] = s->ov[j - 1];
		s->ov[j].line = gl;
		s->ov[j].from = lines[i].replace_from; s->ov[j].to = lines[i].replace_to; s->ov[j].value = lines[i].replace_value;
		s->ov[j].add = NULL;
		if(lines[i].add)
		{
			s->ov[j].add = malloc(sizeof(int16_t) * s->rtab->dp.W);            /* a raster line (pixel rate) */
			memcpy(s->ov[j].add, lines[i].add, sizeof(int16_t) * s->rtab->dp.W);
		}
		s->nov++;
	}
}

static int send_overlays(htv_t *s, long long end_line)
{
	long long line[2048];
	int from[2048], to[2048], value[2048], i, n = 0;
	const int16_t *add[2048];
	for(i = 0; i < s->nov && s->ov[i].line < end_line && n < 2048; i++, n++)
	{
		line[n] = s->ov[i].line; from[n] = s->ov[i].from; to[n] = s->ov[i].to; value[n] = s->ov[i].value;
		add[n] = s->ov[i].add;
	}
	return(htv_dev_set_overlays(s->rdev, n, line, from, to, value, add));
}

/* New pictures for slots slot .. slot + n - 1: from device memory converted in place (k_ingest), from host memory one
 * copy of n pictures that follow each other there, starting at pics[0].data */
static int send_pictures(htv_t *s, int dev, int slot, int n, const htv_device_frame_t *pics, void *stream)
{
	if(dev) return(htv_dev_ingest_frames(s->rdev, slot, n, pics, stream));
	return(htv_dev_upload_frames(s->rdev, slot, n, (const uint32_t *) pics[0].data, stream));
}

/* One device launch sequence for lines [L0, L0 + n): at most MAX_NEW_FRAMES new pictures */
static int render_chunk(htv_t *s, int *pn, int16_t *d_out, int add, void *stream)
{
	int n = *pn, nnew = 0;
	const htv_dparams_t *dp = &s->tab->dp, *rdp = &s->rtab->dp;
	const int64_t L0 = s->next_line;
	/* the frame map starts at the frame of line L0 - 2: lines L0 - 2 .. L0 - 1 are rasterised again as the left
	 * neighbours of this launch (below), and where L0 opens a frame they are lines of the previous frame, with its
	 * picture (the progressive 525-line raster shows a source row on its last line, and the video filter reaches back
	 * into it from line 1) */
	const int64_t fm = (L0 >= 2 ? L0 - 2 : 0) / s->lines, f0 = L0 / s->lines, f1 = (L0 + n - 1) / s->lines;
	int32_t map[4096];
	int64_t f;
	int r, nmap = 0, run_n = 0, run_slot = 0, run_dev = 0;
	htv_device_frame_t run[HTV_INGEST_MAX];       /* the pictures of the run of new ones not sent yet */
	const size_t fpix = (size_t) rdp->active_width * rdp->active_lines;
	void *up, *rup;

	if(f1 - fm + 1 > 4096) return(HTV_ERROR);
	/* frame f0 - 1 was pulled by the previous call, which showed its picture: that call's last slot, or the one before
	 * it where that call also pulled frame f0. Its slot is not reused before this launch has run (the slots cycle
	 * through 16 and a call brings at most MAX_NEW_FRAMES), and its phase of the composite store is already converted */
	if(fm < f0) map[nmap++] = s->cur_frame == f0 ? s->prev_slot : s->cur_slot;

	/* pictures and PCM go up on the encoder's own upload stream, ahead of the kernels queued on
	 * `stream` for the previous chunk and beside the caller's device-to-host copies */
	/* an error between uploads_begin and uploads_end still joins the upload stream(s) back in */
#define UP_FAIL(code) do { htv_dev_uploads_end(s->dev, stream); if(s->rdev != s->dev) htv_dev_uploads_end(s->rdev, stream); return(code); } while(0)
	up = htv_dev_uploads_begin(s->dev);
	rup = s->rdev != s->dev ? htv_dev_uploads_begin(s->rdev) : up;
	/* lines L0 - 2 .. L0 - 1 are rasterised again as the left neighbours of this launch (video / pre-emphasis
	 * filter halo, the resampler's lead, SECAM's chain start): a VBI waveform may reach the last sample of
	 * its line (teletext's raised cosine does, ref teletext.c:1069), so their overlays are still needed */
	drop_overlays_before(s, L0 - 2);

	/* pictures: one pull per frame, at its first line (ref video.c:4873-4881) */
	for(f = f0; f <= f1; f++)
	{
		if(f > s->cur_frame)
		{
			htv_device_frame_t pic;
			int dev = 0, got = 0;
			if(nnew >= MAX_NEW_FRAMES)
			{
				/* every free picture slot is in use by this launch: stop at this frame boundary */
				n = (int) (f * s->lines - L0);
				break;
			}
			if(s->vbi_read && f > f0 && s->nov + MAX_VBI_LINES_PER_FRAME > htv_dev_overlay_capacity())
			{
				/* the overlay table of this launch sequence is full: stop at this frame boundary */
				n = (int) (f * s->lines - L0);
				break;
			}
			memset(&pic, 0, sizeof(pic));
			s->prev_slot = s->cur_slot;
			s->cur_frame = f;
			if(s->av.read_video)
			{
				htv_frame_t fr;
				memset(&fr, 0, sizeof(fr));
				s->dev_read = NULL;                      /* a read_video installed after a device source replaces it */
				got = s->av.read_video(s->av.ctx, &fr) == HTV_OK && fr.framebuffer;
				pic.width = fr.width; pic.height = fr.height; pic.data = fr.framebuffer; pic.serial = fr.serial;
			}
			else if(s->dev_read)
			{
				dev = 1;
				got = s->dev_read(s->dev_ctx, &pic) == HTV_OK && pic.data;
			}
			if(got)
			{
				if(pic.width != rdp->active_width || pic.height != rdp->active_lines)
				{
					fprintf(stderr, "hacktv_b200: source frame is %dx%d, the raster needs %dx%d\n",
						pic.width, pic.height, rdp->active_width, rdp->active_lines);
					UP_FAIL(HTV_ERROR);
				}
				if(!s->have_serial || pic.serial != s->cur_serial || s->cur_slot < 0)
				{
					s->cur_slot = s->next_slot;
					s->next_slot = (s->next_slot + 1) % MAX_FRAME_SLOTS;
					/* new pictures that land in consecutive slots are sent together: from the device as one k_ingest list;
					 * from the host when they follow each other in the caller's memory (a capture ring, htv_av_memory_open's
					 * array), as ONE copy: 2 MB copies beside the 8 MB copies coming back keep neither PCIe direction full */
					if(run_n > 0 && dev == run_dev && s->cur_slot == run_slot + run_n
						&& (dev || (const uint32_t *) pic.data == (const uint32_t *) run[0].data + (size_t) run_n * fpix)) run[run_n++] = pic;
					else
					{
						if(run_n > 0 && (r = send_pictures(s, run_dev, run_slot, run_n, run, rup)) != HTV_OK) UP_FAIL(r);
						run[0] = pic; run_slot = s->cur_slot; run_n = 1; run_dev = dev;
					}
					s->cur_serial = pic.serial;
					s->have_serial = 1;
					nnew++;
				}
			}
			else
			{
				s->av.read_video = NULL;
				s->dev_read = NULL;
				s->cur_slot = -1;
			}
			if(s->vbi_read) pull_overlays(s, f);
		}
		map[nmap++] = s->cur_slot;
	}
	if(run_n > 0 && (r = send_pictures(s, run_dev, run_slot, run_n, run, rup)) != HTV_OK) UP_FAIL(r);
	/* sound: everything the audio clock reaches inside this run */
	if(dp->have_fm || dp->have_am || dp->have_nicam)
	{
		const int64_t m1 = (L0 + n) * (int64_t) s->W + dp->shift;
		r = pull_audio(s, fetches_by(m1 - 1, s->tab->rate), up);
		if(r != HTV_OK) UP_FAIL(r);
	}
	if(s->vbi_read || s->nov)
	{
		/* the raster reaches two lines past the last one emitted: the video filter looks one line ahead, and with
		 * --pixelrate emitted line t is resampled from raster lines t and t + 1 */
		r = send_overlays(s, L0 + n + 2);
		if(r != HTV_OK) UP_FAIL(r);
	}
#undef UP_FAIL
	r = htv_dev_uploads_end(s->dev, stream);
	if(r != HTV_OK) return(r);
	if(s->rdev != s->dev)
	{
		r = htv_dev_uploads_end(s->rdev, stream);
		if(r != HTV_OK) return(r);
	}

	r = htv_dev_set_frame_map(s->rdev, map, nmap, fm, stream);
	if(r != HTV_OK) return(r);

	if(dp->have_fm || dp->have_am || dp->have_nicam)
	{
		const int64_t m0 = L0 * s->W + dp->shift, m1 = (L0 + n) * (int64_t) s->W + dp->shift;
		int64_t mm0 = m0;
		if(L0 == 0) mm0 = 0;      /* the audio clock starts `shift` samples before the first emitted sample */
		r = htv_dev_audio_prepass(s->dev, mm0, m1, stream);
		if(r != HTV_OK) return(r);
	}

	{
		const int16_t *acc = add ? d_out : NULL;
		int acc_lines = add ? n : 0;
		if(s->pt_read)
		{
			if(add) return(HTV_ERROR);                        /* one combiner input at a time */
			acc_lines = pull_passthru(s, n, stream);
			if(acc_lines < 0) return(HTV_ERROR);
			acc = s->pt_dev;
		}
		r = htv_dev_render_lines(s->dev, s->rdev != s->dev ? s->rdev : NULL, L0, n, d_out, acc, acc_lines, stream);
		if(r != HTV_OK) return(r);
	}
	s->next_line += n;
	*pn = n;
	return(HTV_OK);
}

static int max_chunk_lines(const htv_t *s)
{
	/* bounded by the device-side audio / NICAM rings (htv_kernels.cu) */
	double lines_per_s = (double) s->tab->rate / s->W;
	int n = (int) (lines_per_s * MAX_CHUNK_SECONDS);
	return(n < 1 ? 1 : n);
}

static int render_any(htv_t *s, int nlines, int16_t *d_out, size_t *nsamples, int add, void *cuda_stream)
{
	int done = 0, r, cap, align;
	if(!s || nlines < 0 || !d_out) return(HTV_ERROR);
	/* the widest access the store makes to d_out (and htv_render_add's combiner from it, htv_dev_out_align): four int16
	 * samples in the split and FM-video modulators where 4 | W, else one sample. The sub-batches start whole lines in,
	 * which keeps it */
	align = htv_dev_out_align(s->dev);
	if(((uintptr_t) d_out & (uintptr_t) (align - 1)) != 0)
	{
		fprintf(stderr, "hacktv_b200: the output buffer must be %d-byte aligned\n", align);
		return(HTV_ERROR);
	}
	/* pictures and sound from device memory are read after whatever the caller queued on its stream before this call;
	 * the pictures go into the raster context, the sound into the modulating one (the same one without --pixelrate) */
	if(s->dev_read && !s->av.read_video && (r = htv_dev_mark_call(s->rdev, cuda_stream)) != HTV_OK) return(r);
	if(s->adev_read && !s->av.read_audio && (r = htv_dev_mark_call(s->dev, cuda_stream)) != HTV_OK) return(r);
	cap = max_chunk_lines(s);
	if(s->pt_read && cap > PT_MAX_LINES) cap = PT_MAX_LINES;
	while(done < nlines)
	{
		int n = nlines - done;
		if(n > cap) n = cap;
		if(s->pt_read && n > PT_MAX_LINES) n = PT_MAX_LINES;
		r = render_chunk(s, &n, (int16_t *) ((char *) d_out + (size_t) done * s->W * s->bps), add, cuda_stream);
		if(r != HTV_OK) return(r);
		done += n;
	}
	if(nsamples) *nsamples = (size_t) nlines * s->W;
	return(HTV_OK);
}

int htv_render(htv_t *s, int nlines, int16_t *d_out, size_t *nsamples, void *cuda_stream)
{
	return(render_any(s, nlines, d_out, nsamples, 0, cuda_stream));
}

int htv_render_add(htv_t *s, int nlines, int16_t *d_out, size_t *nsamples, void *cuda_stream)
{
	if(s && s->type != HTV_TYPE_INT16)
	{
		/* the sum wraps in int16; convert it once at the end (htv_convert) */
		fprintf(stderr, "hacktv_b200: htv_render_add sums int16 streams; the sample type is %s (use htv_convert on the sum)\n", htv_st_name(s->type));
		return(HTV_ERROR);
	}
	return(render_any(s, nlines, d_out, nsamples, 1, cuda_stream));
}

int htv_mix_add(int16_t *d_acc, const int16_t *d_in, size_t nvalues, void *cuda_stream)
{
	return(htv_dev_mix_add(d_acc, d_in, nvalues, cuda_stream));
}

/* copy-back granularity: small enough that the first render / last copy (which overlap nothing)
 * stay short, large enough for full PCIe rate */
#define HOST_PIECE_BYTES (8u << 20)

/* On an error in the middle of the pipeline both streams are drained before returning, so no
 * asynchronous copy is still writing into the caller's buffer afterwards. */
static int host_fail(htv_t *s, int r)
{
	if(s->st_copy) htv_dev_sync(s->dev, s->st_copy);
	if(s->st_compute) htv_dev_sync(s->dev, s->st_compute);
	return(r);
}

/* Queue the rendering of the next nlines and their copy into host memory (8 MB pieces, rendering of one piece
 * overlapping the copy of the previous one); returns without waiting. */
static int host_enqueue(htv_t *s, int nlines, int16_t *h_out)
{
	const size_t line_bytes = (size_t) s->W * s->bps;
	size_t piece_bytes = HOST_PIECE_BYTES;
	int piece, done = 0, r, i;
	{
		const char *e = getenv("HTV_HOST_PIECE_MB");                    /* experiment knob (tools/e2e_probe.py) */
		if(e && atoi(e) > 0) piece_bytes = (size_t) atoi(e) << 20;
	}
	piece = (int) (piece_bytes / line_bytes);
	if(piece < 1) piece = 1;
	if(piece > nlines) piece = nlines > 0 ? nlines : 1;
	if((size_t) piece * line_bytes > s->d_stage_bytes)
	{
		if(s->st_copy) { htv_dev_sync(s->dev, s->st_copy); htv_dev_sync(s->dev, s->st_compute); }
		for(i = 0; i < 2; i++)
		{
			htv_dev_free(s->dev, s->d_stage[i]);
			s->d_stage[i] = htv_dev_alloc(s->dev, (size_t) piece * line_bytes);
			if(!s->d_stage[i]) { s->d_stage_bytes = 0; return(HTV_OUT_OF_MEMORY); }
		}
		s->d_stage_bytes = (size_t) piece * line_bytes;
		s->piece_i = 0;
	}
	if(!s->st_compute)
	{
		s->st_compute = htv_dev_stream_new(s->dev);
		s->st_copy = htv_dev_stream_new(s->dev);
		for(i = 0; i < 2; i++)
		{
			s->ev_rendered[i] = htv_dev_event_new(s->dev); s->ev_copied[i] = htv_dev_event_new(s->dev);
			s->ev_frame[i] = htv_dev_event_new(s->dev);
		}
	}
	for(; done < nlines; done += piece, s->piece_i++)
	{
		const int n = nlines - done < piece ? nlines - done : piece, b = s->piece_i & 1;
		/* the staging buffer must have been copied out before it is rendered into again */
		if(s->piece_i >= 2 && (r = htv_dev_stream_wait(s->st_compute, s->ev_copied[b])) != HTV_OK) return(host_fail(s, r));
		r = htv_render(s, n, s->d_stage[b], NULL, s->st_compute);
		if(r != HTV_OK) return(host_fail(s, r));
		if((r = htv_dev_event_record(s->ev_rendered[b], s->st_compute)) != HTV_OK) return(host_fail(s, r));
		if((r = htv_dev_stream_wait(s->st_copy, s->ev_rendered[b])) != HTV_OK) return(host_fail(s, r));
		r = htv_dev_memcpy_d2h(s->dev, (char *) h_out + (size_t) done * line_bytes, s->d_stage[b], (size_t) n * line_bytes, s->st_copy);
		if(r != HTV_OK) return(host_fail(s, r));
		if((r = htv_dev_event_record(s->ev_copied[b], s->st_copy)) != HTV_OK) return(host_fail(s, r));
	}
	return(HTV_OK);
}

int htv_render_host(htv_t *s, int nlines, int16_t *h_out, size_t *nsamples)
{
	int r;
	if(!s || nlines < 0 || !h_out) return(HTV_ERROR);
	/* a frame prefetched for htv_next_line is part of the stream: mixing the two pull styles would reorder it */
	if(s->pf_pending) return(HTV_ERROR);
	r = host_enqueue(s, nlines, h_out);
	if(r != HTV_OK) return(r);
	if(nsamples) *nsamples = (size_t) nlines * s->W;
	r = htv_dev_sync(s->dev, s->st_copy);
	if(r != HTV_OK) return(host_fail(s, r));
	return(htv_dev_sync(s->dev, s->st_compute));
}

int htv_set_prefetch(htv_t *s, int on)
{
	if(!s) return(HTV_ERROR);
	s->prefetch = on != 0;
	return(HTV_OK);
}

/* Start rendering the next frame's worth of lines into h_frame[buf]; htv_next_line collects it later */
static int frame_enqueue(htv_t *s, int buf, int n)
{
	int r;
	s->pf_first_line = s->next_line;
	r = host_enqueue(s, n, s->h_frame[buf]);
	if(r != HTV_OK) return(r);
	r = htv_dev_event_record(s->ev_frame[buf], s->st_copy);
	if(r != HTV_OK) return(host_fail(s, r));
	s->pf_lines = n;
	s->pf_pending = 1;
	return(HTV_OK);
}

htv_line_t *htv_next_line(htv_t *s)
{
	if(!s) return(NULL);
	if(s->type != HTV_TYPE_INT16)
	{
		/* vid_next_line's contract: int16 I,Q lines (the reference's sink converts them) */
		fprintf(stderr, "hacktv_b200: htv_next_line hands out int16 lines; the sample type is %s (use htv_render / htv_render_host)\n", htv_st_name(s->type));
		return(NULL);
	}
	if(s->h_pos >= s->h_lines)
	{
		if(!s->h_frame[0])
		{
			s->h_frame[0] = htv_dev_alloc_pinned((size_t) s->lines * s->W * s->bps);
			s->h_frame[1] = htv_dev_alloc_pinned((size_t) s->lines * s->W * s->bps);
			s->h_iq = malloc(sizeof(int16_t) * 2 * s->W);
			if(!s->h_frame[0] || !s->h_frame[1] || !s->h_iq) return(NULL);
		}
		if(s->pf_pending)
		{
			/* the frame rendered while the caller consumed the previous one */
			if(htv_dev_event_wait(s->ev_frame[s->h_cur ^ 1]) != HTV_OK) return(NULL);
			s->h_cur ^= 1;
			s->h_first_line = s->pf_first_line;
			s->h_lines = s->pf_lines;
			s->pf_pending = 0;
		}
		else
		{
			/* refill: the rest of the current frame (a whole frame in steady state) */
			const int n = s->lines - (int) (s->next_line % s->lines);
			s->h_first_line = s->next_line;
			if(htv_render_host(s, n, s->h_frame[s->h_cur], NULL) != HTV_OK) return(NULL);
			s->h_lines = n;
		}
		s->h_pos = 0;
		/* htv_set_prefetch: the next frame starts its way through the GPU and the copy engine now; it pulls its
		 * picture and sound from the source one frame earlier than the reference would */
		if(s->prefetch && frame_enqueue(s, s->h_cur ^ 1, s->lines - (int) (s->next_line % s->lines)) != HTV_OK) return(NULL);
	}
	{
		const int64_t L = s->h_first_line + s->h_pos;
		int16_t *src = s->h_frame[s->h_cur] + (size_t) s->h_pos * s->W * (s->complex ? 2 : 1);
		if(s->complex) s->line.output = src;
		else
		{
			int x;
			for(x = 0; x < s->W; x++) { s->h_iq[x * 2] = src[x]; s->h_iq[x * 2 + 1] = 0; }
			s->line.output = s->h_iq;
		}
		s->line.width = s->W;
		s->line.frame = (int) (L / s->lines) + 1;
		s->line.line = (int) (L % s->lines) + 1;
		s->h_pos++;
	}
	return(&s->line);
}
