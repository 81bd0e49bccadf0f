/* A plain-C consumer of include/midi_b200.h (no CUDA headers, no Python): proves that the boundary is a C ABI a maintainer can
 * bind from any host language.  Runs WITHOUT a GPU: only entry points that do not launch are called -- the version / size
 * queries and the argument validation that precedes every launch (error code + thread-local message). */
#include <stdio.h>
#include <string.h>
#include "midi_b200.h"

int main(void) {
    int fails = 0;
    if (b200_abi_version() != 1) { printf("abi_version %d\n", b200_abi_version()); fails++; }
    if (b200_decode_desc_bytes() != sizeof(b200_decode_desc)) { printf("decode_desc size mismatch\n"); fails++; }
    /* split-K workspace: splits * M * N fp32 partials */
    if (b200_gemm_workspace_bytes(1024, 1024, 4) != (size_t)4 * 1024 * 1024 * sizeof(float)) { printf("workspace bytes\n"); fails++; }
    /* accumulate without split-K still reduces through one fp32 slice: the query covers it */
    if (b200_gemm_workspace_bytes(300, 520, 1) != (size_t)300 * 520 * sizeof(float)) { printf("workspace bytes, splits 1\n"); fails++; }
    /* argument validation happens before any CUDA call: an empty problem is B200_ERR_ARG with a message */
    int rc = b200_gemm_bf16(NULL, NULL, NULL, NULL, 0, 0, 0, 8, 8, 8, 0, 0, 0, 0, 128, 1, NULL, 0, NULL);
    if (rc != B200_ERR_ARG) { printf("empty gemm: rc %d\n", rc); fails++; }
    if (strstr(b200_last_error(), "gemm") == NULL) { printf("last_error: '%s'\n", b200_last_error()); fails++; }
    /* unaligned leading dimension */
    rc = b200_gemm_bf16((void*)256, (void*)256, (void*)256, NULL, 128, 128, 64, 63, 64, 128, 0, 0, 0, 0, 128, 1, NULL, 0, NULL);
    if (rc != B200_ERR_ARG) { printf("lda=63: rc %d\n", rc); fails++; }
    rc = b200_swiglu_fwd(NULL, NULL, 4, 12, NULL);         /* intermediate size not a multiple of 8 */
    if (rc != B200_ERR_ARG) { printf("swiglu I=12: rc %d\n", rc); fails++; }
    rc = b200_scale_bf16((void*)2, (void*)16, 8, 2.0f, NULL);   /* misaligned operand */
    if (rc != B200_ERR_ARG) { printf("scale misaligned: rc %d\n", rc); fails++; }
    printf(fails ? "FAILED %d\n" : "abi host ok\n", fails);
    return fails;
}
