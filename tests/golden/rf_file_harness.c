/* The reference's own file sink writers (ref rf_file.c, rf.c), linked unmodified from the objects the oracle build
 * compiles in place, fed every int16 value: 65 536 complex samples I = k - 32768, Q = ~I (k = 0 .. 65535), through
 * each of the twelve writers (six types x complex / real). Writes <dir>/<type>_<complex|real>.bin.
 * Built and run by tests/golden/make_golden_sample_types.py, which pins the streams' sizes and sha256. */
#include <stdio.h>
#include <stdint.h>
#include "rf.h"

int main(int argc, char **argv)
{
	static const char *const names[] = { "uint8", "int8", "uint16", "int16", "int32", "float" };
	static int16_t iq[65536 * 2];
	char path[4096];
	int k, type, cpx;
	if(argc < 2) { fprintf(stderr, "usage: rf_file_harness <dir>\n"); return(2); }
	for(k = 0; k < 65536; k++) { iq[2 * k] = (int16_t) (k - 32768); iq[2 * k + 1] = (int16_t) ~iq[2 * k]; }
	for(type = RF_UINT8; type <= RF_FLOAT; type++)
	{
		for(cpx = 1; cpx >= 0; cpx--)
		{
			rf_t rf;
			snprintf(path, sizeof(path), "%s/%s_%s.bin", argv[1], names[type], cpx ? "complex" : "real");
			if(rf_file_open(&rf, path, type, cpx) != RF_OK) return(1);
			if(rf_write(&rf, iq, 65536) != RF_OK) return(1);
			rf_close(&rf);
		}
	}
	return(0);
}
