/* CPU check of the sample-type conversion (hacktv_b200/csrc/htv_sample_type.h), the same functions the device stores
 * run: 65 536 complex samples I = k - 32768, Q = ~I (k = 0 .. 65535) written as each of the twelve streams (six types x
 * complex / real) the reference's file sink writes, with htv_st_put2 (complex) and htv_st_put (real, I only).
 * Writes <dir>/<type>_<complex|real>.bin; tests/test_sample_type_host.py compares them with the pinned digests. */
#include <stdio.h>
#include <stdlib.h>
#include "htv_sample_type.h"

int main(int argc, char **argv)
{
	static int16_t iq[65536 * 2];
	static uint8_t out[65536 * 2 * 4];
	char path[4096];
	int k, type, cpx;
	if(argc < 2) { fprintf(stderr, "usage: sample_type_emu <dir>\n"); return(2); }
	for(k = 0; k < 65536; k++) { iq[2 * k] = (int16_t) (k - 32768); iq[2 * k + 1] = (int16_t) ~iq[2 * k]; }
	for(type = HTV_TYPE_UINT8; type <= HTV_TYPE_FLOAT; type++)
	{
		for(cpx = 1; cpx >= 0; cpx--)
		{
			FILE *f;
			for(k = 0; k < 65536; k++)
			{
				if(cpx) htv_st_put2(out, (size_t) k, type, iq[2 * k], iq[2 * k + 1]);
				else htv_st_put(out, (size_t) k, type, iq[2 * k]);
			}
			snprintf(path, sizeof(path), "%s/%s_%s.bin", argv[1], htv_st_name(type), cpx ? "complex" : "real");
			f = fopen(path, "wb");
			if(!f || fwrite(out, (size_t) htv_st_bytes(type, cpx), 65536, f) != 65536) return(1);
			fclose(f);
		}
	}
	return(0);
}
