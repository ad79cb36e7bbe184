/*
 * simplegrep_b200.c -- the reference's simplegrep example flow
 * (examples/simplegrep.c:173-215: hs_compile -> hs_alloc_scratch -> hs_scan with
 * an event handler that prints the end offset -> hs_free_*), written against
 * include/hs_b200.h and linked with libhs_b200.so instead of libhs.  Config 1 of
 * BASELINE.json ("simplegrep: 1 literal pattern, 1 MB ASCII buffer, block mode").
 *
 *   cc -O2 -o simplegrep_b200 examples/simplegrep_b200.c -Iinclude \
 *      -Lhyperscan_b200/lib -lhs_b200 -Wl,-rpath,$PWD/hyperscan_b200/lib
 *   ./simplegrep_b200 <pattern> <input file>
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "hs_b200.h"

static int eventHandler(unsigned int id, unsigned long long from, unsigned long long to,
                        unsigned int flags, void *ctx) {
    (void)id;
    (void)from;
    (void)flags;
    printf("Match for pattern \"%s\" at offset %llu\n", (const char *)ctx, to);
    return 0;
}

static char *readInputData(const char *path, unsigned int *length) {
    FILE *f = fopen(path, "rb");
    if (!f) {
        fprintf(stderr, "ERROR: unable to open file \"%s\"\n", path);
        return NULL;
    }
    fseek(f, 0, SEEK_END);
    long n = ftell(f);
    fseek(f, 0, SEEK_SET);
    char *buf = malloc(n > 0 ? (size_t)n : 1);
    if (!buf || (n > 0 && fread(buf, 1, (size_t)n, f) != (size_t)n)) {
        fprintf(stderr, "ERROR: unable to read input\n");
        fclose(f);
        free(buf);
        return NULL;
    }
    fclose(f);
    *length = (unsigned int)n;
    return buf;
}

int main(int argc, char *argv[]) {
    if (argc != 3) {
        fprintf(stderr, "Usage: %s <pattern> <input file>\n", argv[0]);
        return -1;
    }
    char *pattern = argv[1];
    hs_database_t *database;
    hs_compile_error_t *compile_err;
    if (hs_compile(pattern, HS_FLAG_DOTALL, HS_MODE_BLOCK, NULL, &database, &compile_err) != HS_SUCCESS) {
        fprintf(stderr, "ERROR: Unable to compile pattern \"%s\": %s\n", pattern, compile_err->message);
        hs_free_compile_error(compile_err);
        return -1;
    }
    unsigned int length;
    char *inputData = readInputData(argv[2], &length);
    if (!inputData) {
        hs_free_database(database);
        return -1;
    }
    hs_scratch_t *scratch = NULL;
    hs_error_t rc = hs_alloc_scratch(database, &scratch);
    if (rc != HS_SUCCESS) {
        fprintf(stderr, "ERROR: Unable to allocate scratch space (%d)%s. Exiting.\n", rc,
                rc == HS_ARCH_ERROR ? ": no usable CUDA device, and there is no CPU scan path" : "");
        free(inputData);
        hs_free_database(database);
        return -1;
    }
    printf("Scanning %u bytes with Hyperscan (H100 runtime %s)\n", length, hs_version());
    if (hs_scan(database, inputData, length, 0, scratch, eventHandler, pattern) != HS_SUCCESS) {
        fprintf(stderr, "ERROR: Unable to scan input buffer. Exiting.\n");
        hs_free_scratch(scratch);
        free(inputData);
        hs_free_database(database);
        return -1;
    }
    hs_free_scratch(scratch);
    free(inputData);
    hs_free_database(database);
    return 0;
}
