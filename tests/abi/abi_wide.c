/* A plain-C consumer of the persistent generate kernel's batch limits (no CUDA headers): the per-request entry
 * b200_decode_events_queue_rows takes 1..32 rows and the plain entry b200_decode_events 1..16.  A descriptor that fails a
 * later check (hidden 0) shows which batches pass the batch check, before any CUDA call, so this runs without a GPU. */
#include <stdio.h>
#include <string.h>
#include "midi_b200.h"

static int rows_call(b200_decode_desc* d) {
    int off = 0, end = 0, last = 0, top_k = 1, first = 0;
    float temp = 1.f, top_p = 1.f;
    unsigned long long seed = 0;
    return b200_decode_events_queue_rows(d, &off, &end, &last, 0, 1, NULL, 0, &temp, &top_p, &top_k, &seed, &first, NULL);
}

static int expect(int rc, const char* what, const char* msg) {
    if (rc != B200_ERR_ARG || strstr(b200_last_error(), msg) == NULL) {
        printf("%s: rc %d, last_error '%s' (want '%s')\n", what, rc, b200_last_error(), msg);
        return 1;
    }
    return 0;
}

int main(void) {
    int fails = 0;
    b200_decode_desc d;
    memset(&d, 0, sizeof d);
    d.batch = 33;
    fails += expect(rows_call(&d), "rows batch 33", "batch 33 outside 1..32");
    d.batch = 32;
    fails += expect(rows_call(&d), "rows batch 32", "hidden 1024");
    d.batch = 17;
    fails += expect(rows_call(&d), "rows batch 17", "hidden 1024");
    fails += expect(b200_decode_events(&d, 1, NULL, 0, NULL), "plain batch 17", "batch 17 outside 1..16");
    d.batch = 16;
    fails += expect(b200_decode_events(&d, 1, NULL, 0, NULL), "plain batch 16", "hidden 1024");
    printf(fails ? "FAILED %d\n" : "abi wide ok\n", fails);
    return fails;
}
