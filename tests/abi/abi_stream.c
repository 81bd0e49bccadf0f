/* A plain-C consumer of b200_decode_events_queue_stream (no CUDA headers): without its pinned host buffers the entry
 * refuses with B200_ERR_ARG and a message, before any CUDA call, so this runs without a GPU. */
#include <stdio.h>
#include <string.h>
#include "midi_b200.h"

int main(void) {
    int fails = 0;
    b200_decode_desc d;
    long long out[8];
    int committed = 0, ctl = 0;
    memset(&d, 0, sizeof d);
    int rc = b200_decode_events_queue_stream(&d, NULL, NULL, NULL, 0, 1, NULL, 0, NULL, NULL, NULL, NULL, NULL, NULL,
                                             &committed, &ctl, NULL);
    if (rc != B200_ERR_ARG) { printf("no out_events: rc %d\n", rc); fails++; }
    if (strstr(b200_last_error(), "out_events") == NULL) { printf("last_error: '%s'\n", b200_last_error()); fails++; }
    rc = b200_decode_events_queue_stream(&d, NULL, NULL, NULL, 0, 1, NULL, 0, NULL, NULL, NULL, NULL, NULL, out, &committed,
                                         NULL, NULL);
    if (rc != B200_ERR_ARG) { printf("no ctl: rc %d\n", rc); fails++; }
    printf(fails ? "FAILED %d\n" : "abi stream ok\n", fails);
    return fails;
}
