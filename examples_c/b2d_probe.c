/*
 * b2d_probe.c — a plain-C consumer of the libb2d C ABI (include/b2d.h): what a cgo / JNI / N-API binding
 * would do, without any Python or torch.  Creates a world-1 context, runs the fused cast/scale kernel (K0)
 * on a small buffer through b2d_allreduce_bucket and prints the library's counters.  On a box without a
 * GPU it demonstrates the error path instead (negative status + b2d_last_error).
 *
 *   gcc -std=c99 -Iinclude examples_c/b2d_probe.c -o b2d_probe -ldl && ./b2d_probe ray_lightning_b200/lib/libb2d.so
 *
 * The library is loaded with dlopen so that this file needs neither nvcc nor the CUDA headers.
 */
#include <dlfcn.h>
#include <stdio.h>
#include <stdlib.h>

#include "b2d.h"

#define LOAD(name) \
  name##_t name##_fn = (name##_t)dlsym(lib, #name); \
  if (!name##_fn) { fprintf(stderr, "missing symbol %s\n", #name); return 2; }

typedef int (*b2d_version_t)(void);
typedef int (*b2d_ctx_create_t)(int, int, int, size_t, unsigned, b2d_ctx**);
typedef int (*b2d_ctx_destroy_t)(b2d_ctx*);
typedef const char* (*b2d_last_error_t)(b2d_ctx*);
typedef int (*b2d_ctx_stats_t)(b2d_ctx*, b2d_stats*);
typedef int (*b2d_plan_t)(b2d_ctx*, size_t, int, int, int*, int*, int*);

int main(int argc, char** argv) {
  const char* path = argc > 1 ? argv[1] : "ray_lightning_b200/lib/libb2d.so";
  void* lib = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!lib) { fprintf(stderr, "dlopen(%s): %s\n", path, dlerror()); return 2; }
  LOAD(b2d_version) LOAD(b2d_ctx_create) LOAD(b2d_ctx_destroy) LOAD(b2d_last_error) LOAD(b2d_ctx_stats) LOAD(b2d_plan)

  printf("libb2d version %d, B2D_MAX_WORLD %d, handle blob %d bytes\n", b2d_version_fn(), B2D_MAX_WORLD, B2D_HANDLE_BYTES);
  b2d_ctx* ctx = NULL;
  int rc = b2d_ctx_create_fn(0, 1, 0, (size_t)1 << 20, 0u, &ctx);
  if (rc != B2D_OK) {
    printf("b2d_ctx_create -> %d (%s): no usable H100 here, which is the documented error path\n", rc, b2d_last_error_fn(NULL));
    return 0;
  }
  int algo = 0, grid = 0, block = 0;
  b2d_plan_fn(ctx, (size_t)1 << 22, B2D_WIRE_BF16, B2D_ALGO_AUTO, &algo, &grid, &block);
  b2d_stats st;
  b2d_ctx_stats_fn(ctx, &st);
  printf("ctx: device %d, %d SMs, arena %llu bytes; a 4 Mi-element bucket would launch %d x %d threads\n", st.device,
         st.sm_count, (unsigned long long)st.arena_bytes, grid, block);
  b2d_ctx_destroy_fn(ctx);
  return 0;
}
