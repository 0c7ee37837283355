/* htv_cli - a small front end with hacktv's calling sequence (ref hacktv.c:1440-1601):
 *
 *     htv_cli -m i -s 16000000 --filter -o out.bin [-t int8] [--lines N] test
 *
 * mode lookup -> config overrides (ref hacktv.c:1107-1437, in-scope options only) ->
 * htv_init -> test source -> { htv_next_line; htv_rf_write } -> close. It exists to show
 * the C-ABI driven exactly as the reference drives video.h, and to produce files that
 * can be compared byte-for-byte with `hacktv -o file [-t type]`. For a sample type other
 * than int16 the encoder converts on the device and the file is written from
 * htv_render_host, up to one frame per call.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <signal.h>
#include "hacktv_b200.h"

static const char *const _types[] = { "uint8", "int8", "uint16", "int16", "int32", "float" };   /* HTV_TYPE_* */

static volatile sig_atomic_t _abort = 0;
static void on_signal(int sig) { (void) sig; _abort = 1; }

static void usage(void)
{
	fprintf(stderr,
		"Usage: htv_cli [options] test\n"
		"  -m, --mode <name>      TV mode (default: i). --list-modes prints them\n"
		"  -s, --samplerate <hz>  Sample rate (default: 16000000)\n"
		"  -o, --output <file>    Output file, '-' for stdout (IQ or real)\n"
		"  -t, --type <type>      Sample type: uint8, int8, uint16, int16 (default), int32, float\n"
		"      --filter           Enable the VSB / low-pass video filter\n"
		"      --nocolour --noaudio --nonicam --swap-iq\n"
		"      --s-video          Chroma on Q, luma on I (PAL, SECAM or NTSC baseband modes; the file is I,Q)\n"
		"      --offset <hz>  --level <f>  --volume <f>\n"
		"      --lines <n>        Stop after n scan lines (default: run until interrupted)\n");
}

int main(int argc, char **argv)
{
	const char *mode = "i", *out = NULL, *input = NULL;
	unsigned int rate = 16000000, pixelrate = 0;   /* --pixelrate: raster at this rate, resampled to -s (not yet run on a GPU) */
	int filter = 0, nocolour = 0, noaudio = 0, nonicam = 0, swap_iq = 0, s_video = 0, type = HTV_TYPE_INT16, i;
	long long offset = 0, lines = -1, n = 0;
	double level = 1.0, volume = 1.0;
	const htv_config_t *mc;
	htv_config_t conf;
	htv_t *vid = NULL;
	htv_rf_t rf;

	for(i = 1; i < argc; i++)
	{
		const char *a = argv[i];
		if((!strcmp(a, "-m") || !strcmp(a, "--mode")) && i + 1 < argc) mode = argv[++i];
		else if((!strcmp(a, "-s") || !strcmp(a, "--samplerate")) && i + 1 < argc) rate = strtoul(argv[++i], NULL, 10);
		else if(!strcmp(a, "--pixelrate") && i + 1 < argc) pixelrate = strtoul(argv[++i], NULL, 10);
		else if((!strcmp(a, "-o") || !strcmp(a, "--output")) && i + 1 < argc) out = argv[++i];
		else if((!strcmp(a, "-t") || !strcmp(a, "--type")) && i + 1 < argc)
		{
			const char *t = argv[++i];
			for(type = 0; type < 6 && strcmp(t, _types[type]); type++);
			if(type == 6) { fprintf(stderr, "Unrecognised file data type.\n"); return(-1); }
		}
		else if(!strcmp(a, "--filter")) filter = 1;
		else if(!strcmp(a, "--nocolour") || !strcmp(a, "--nocolor")) nocolour = 1;
		else if(!strcmp(a, "--noaudio")) noaudio = 1;
		else if(!strcmp(a, "--nonicam")) nonicam = 1;
		else if(!strcmp(a, "--swap-iq")) swap_iq = 1;
		else if(!strcmp(a, "--s-video")) s_video = 1;
		else if(!strcmp(a, "--offset") && i + 1 < argc) offset = strtoll(argv[++i], NULL, 10);
		else if(!strcmp(a, "--level") && i + 1 < argc) level = atof(argv[++i]);
		else if(!strcmp(a, "--volume") && i + 1 < argc) volume = atof(argv[++i]);
		else if(!strcmp(a, "--lines") && i + 1 < argc) lines = strtoll(argv[++i], NULL, 10);
		else if(!strcmp(a, "--list-modes"))
		{
			const htv_mode_t *m;
			for(m = htv_modes; m->id; m++) printf("  %-14s = %s\n", m->id, m->desc);
			return(0);
		}
		else if(a[0] == '-' && a[1]) { usage(); return(-1); }
		else input = a;
	}

	if(!input) { fprintf(stderr, "No input specified.\n"); return(-1); }
	if(strcmp(input, "test") != 0) { fprintf(stderr, "Only the 'test' source is built into htv_cli.\n"); return(-1); }

	mc = htv_find_mode(mode);
	if(!mc) { fprintf(stderr, "Unrecognised TV mode.\n"); return(-1); }
	memcpy(&conf, mc, sizeof(conf));

	if(nocolour && (conf.colour_mode == HTV_PAL || conf.colour_mode == HTV_SECAM || conf.colour_mode == HTV_NTSC))
	{
		conf.colour_mode = HTV_MONOCHROME;
	}
	if(s_video)
	{
		/* ref hacktv.c:1136-1148 */
		if((conf.colour_mode != HTV_PAL && conf.colour_mode != HTV_SECAM && conf.colour_mode != HTV_NTSC) ||
		   conf.output_type != HTV_INT16_REAL)
		{
			fprintf(stderr, "S-Video is only available with PAL, SECAM, or NTSC baseband modes.\n");
			return(-1);
		}
		conf.s_video = 1;
	}
	if(noaudio)
	{
		conf.fm_mono_level = conf.am_audio_level = conf.nicam_level = 0;
		conf.fm_mono_carrier = conf.nicam_carrier = conf.am_mono_carrier = 0;
	}
	if(nonicam) { conf.nicam_level = 0; conf.nicam_carrier = 0; }
	conf.level *= (float) level;
	if(filter) conf.vfilter = 1;
	conf.swap_iq = swap_iq;
	conf.offset = offset;
	conf.volume = (float) volume * 256 + 0.5;

	signal(SIGINT, on_signal);
	signal(SIGTERM, on_signal);
	signal(SIGPIPE, on_signal);

	if(htv_init(&vid, rate, pixelrate, &conf) != HTV_OK)
	{
		fprintf(stderr, "Unable to initialise video encoder.\n");
		return(-1);
	}
	htv_info(vid);

	if(type != HTV_TYPE_INT16)
	{
		/* the device writes the type; the file gets the bytes as they come back */
		FILE *f;
		char *buf;
		const int per_frame = htv_lines_per_frame(vid);
		size_t line_bytes;
		int r = 0;
		if(htv_set_sample_type(vid, type) != HTV_OK) { htv_free(vid); return(-1); }
		line_bytes = (size_t) htv_samples_per_line(vid) * htv_bytes_per_sample(vid);   /* of the type just set */
		if(out == NULL) { fprintf(stderr, "No output filename provided.\n"); htv_free(vid); return(-1); }
		f = strcmp(out, "-") == 0 ? stdout : fopen(out, "wb");
		if(!f) { perror("fopen"); htv_free(vid); return(-1); }
		buf = malloc((size_t) per_frame * line_bytes);
		if(buf && htv_av_test_open(htv_av(vid)) == HTV_OK)
		{
			while(!_abort && (lines < 0 || n < lines))
			{
				const int k = lines >= 0 && lines - n < per_frame ? (int) (lines - n) : per_frame;
				if(htv_render_host(vid, k, (int16_t *) buf, NULL) != HTV_OK) { r = -1; break; }
				if(fwrite(buf, line_bytes, (size_t) k, f) != (size_t) k) break;
				n += k;
			}
		}
		free(buf);
		if(f != stdout) fclose(f);
		else fflush(f);
		htv_free(vid);
		fprintf(stderr, "\n");
		return(r);
	}

	if(htv_rf_file_open(&rf, out, htv_is_complex(vid)) != HTV_OK)
	{
		htv_free(vid);
		return(-1);
	}

	if(htv_av_test_open(htv_av(vid)) == HTV_OK)
	{
		htv_set_prefetch(vid, 1);                          /* the test source never ends */
		while(!_abort && (lines < 0 || n < lines))
		{
			htv_line_t *line = htv_next_line(vid);
			if(line == NULL) break;
			if(htv_rf_write(&rf, line->output, line->width) != HTV_OK) break;
			n++;
		}
	}

	htv_rf_close(&rf);
	htv_free(vid);
	fprintf(stderr, "\n");
	return(0);
}
