/* k_line's per-lane sound feed (hacktv_b200/csrc/htv_line.cuh KlFeed) on the CPU: a lane's audio-clock index m grows
 * by W per line, and the feed advances the quotients and remainders of its sound state by the increments of one line
 * (htv_dparams_t kl_w_*, set in htv_dev_create). This checks, line by line, that the advanced state equals the closed
 * forms computed directly from m:
 *   audio:  32000 (m + 1) = aq rate + ar   (j = aq - 1; the segment started ar / 32000 samples ago, the next starts
 *           ceil((rate - ar) / 32000) samples on)
 *   NICAM:  m D = sq F + sr                (s = sq; ceil(s F / D) = m - sr / D; s + 1 starts ceil((F - sr) / D) on)
 *   kk = m mod 32767, cc = m mod cc_len
 * usage: sound_feed_emu rate W shift line0 nlines  -> "OK <lines> <lanes>" or the first mismatch */
#include <stdio.h>
#include <stdlib.h>
#include <stdint.h>

typedef unsigned long long u64;

static u64 gcd64(u64 a, u64 b) { while(b) { u64 t = a % b; a = b; b = t; } return(a); }

/* first audio-clock sample of the segment of audio index j (>= -1) and first sample of NICAM symbol s, as the device's
 * seg_start and nic_sym_pos */
static long long seg_start(long long j, u64 rate) { return(j < 0 ? 0 : (long long) (((u64) (j + 1) * rate + 31999) / 32000) - 1); }
static long long sym_pos(u64 s, u64 F, u64 D) { return((long long) ((s * F + D - 1) / D)); }

int main(int argc, char **argv)
{
	if(argc < 6) return(2);
	const u64 rate = strtoull(argv[1], NULL, 10);
	const int W = atoi(argv[2]), shift = atoi(argv[3]);
	const long long line0 = atoll(argv[4]);
	const int nlines = atoi(argv[5]);
	const u64 g = gcd64(rate, 364000), F = rate / g, D = 364000 / g;
	const u64 cc_len = rate / gcd64(rate, 6552000);      /* the carrier period of the NICAM carrier at 6.552 MHz */
	/* one line's increments (htv_dev_create) */
	const unsigned w_kk = W % 32767, w_cc = (unsigned) (W % cc_len);
	const unsigned w_aq = (unsigned) ((u64) W * 32000 / rate), w_ar = (unsigned) ((u64) W * 32000 % rate);
	const unsigned w_sq = (unsigned) ((u64) W * D / F), w_sr = (unsigned) ((u64) W * D % F);
	int lanes = 0;
	for(int xb = 0; xb < W; xb += 8, lanes++)
	{
		long long m = line0 * W + shift + xb;
		/* set-up by exact division, as kl_feed_init */
		unsigned kk = (unsigned) (m % 32767), cc = (unsigned) ((u64) m % cc_len);
		unsigned aq = (unsigned) ((u64) (m + 1) * 32000 / rate), ar = (unsigned) ((u64) (m + 1) * 32000 % rate);
		unsigned sq = (unsigned) ((u64) m * D / F), sr = (unsigned) ((u64) m * D % F);
		for(int l = 0; l < nlines; l++, m += W)
		{
			const long long j = (long long) ((u64) (m + 1) * 32000 / rate) - 1;
			const u64 s = (u64) m * D / F;
			const long long st = seg_start(j, rate), nx = seg_start(j + 1, rate);
			/* the segment start as kl_lane_feed uses it: m - floor(ar / 32000), one less for j = -1 (its record is stored one
			 * angle step back) */
			const long long st_feed = m - ar / 32000 + (j < 0 ? 1 : 0);
			const long long nb_feed = (long long) ((rate - ar + 31999) / 32000);
			const long long ps = sym_pos(s, F, D), pn = sym_pos(s + 1, F, D);
			const int bad = kk != (unsigned) (m % 32767) || cc != (unsigned) ((u64) m % cc_len) ||
				aq != (unsigned) (j + 1) || st_feed != st || m + nb_feed != nx ||
				sq != (unsigned) s || m - (long long) (sr / D) != ps || m + (long long) ((F - sr + D - 1) / D) != pn;
			if(bad)
			{
				printf("MISMATCH rate %llu W %d lane %d line %lld m %lld: kk %u cc %u aq %u (j %lld) st %lld/%lld nb %lld/%lld "
					"sq %u (s %llu) pos %lld/%lld next %lld/%lld\n", rate, W, xb, line0 + l, m, kk, cc, aq, j, st_feed, st,
					m + nb_feed, nx, sq, s, m - (long long) (sr / D), ps, m + (long long) ((F - sr + D - 1) / D), pn);
				return(1);
			}
			/* W samples on, as kl_feed_next */
			kk += w_kk; if(kk >= 32767) kk -= 32767;
			aq += w_aq; ar += w_ar; if(ar >= rate) { ar -= (unsigned) rate; aq++; }
			sq += w_sq; sr += w_sr; if(sr >= F) { sr -= (unsigned) F; sq++; }
			cc += w_cc; if(cc >= cc_len) cc -= (unsigned) cc_len;
		}
	}
	printf("OK %d %d\n", nlines, lanes);
	return(0);
}
