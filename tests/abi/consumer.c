/* A torch-free consumer of the drop-in boundary: include/b200ddp.h must compile as strict C99, and every declared entry
 * point must resolve from libb200ddp.so with plain dlopen/dlsym.  The calls made here are argument-validation paths only
 * (they return B2_EINVAL before touching CUDA), so the program also runs on a host without a GPU.
 * Built and run by tests/test_abi.py; exit code 0 = all checks passed. */
#include <dlfcn.h>
#include <stdio.h>
#include <string.h>

#include "b200ddp.h"

#define CHECK(cond)                                                      \
  do {                                                                   \
    if (!(cond)) {                                                       \
      fprintf(stderr, "consumer.c:%d: check failed: %s\n", __LINE__, #cond); \
      return 1;                                                          \
    }                                                                    \
  } while (0)

typedef int (*version_fn)(void);
typedef const char* (*last_error_fn)(void);
typedef int (*allreduce_fn)(b2_comm_t*, void*, size_t, int, float, int, void*);
typedef int (*destroy_fn)(b2_comm_t*);
typedef int (*auto_algo_fn)(int, int, size_t, int);
typedef int (*set_param_fn)(b2_comm_t*, const char*, long long);
typedef uint64_t (*op_count_fn)(const b2_comm_t*);

int main(int argc, char** argv) {
  static const char* const symbols[] = {B2_CONSUMER_SYMBOLS};
  void* lib;
  size_t i;
  version_fn version;
  last_error_fn last_error;
  allreduce_fn allreduce;
  destroy_fn destroy;
  auto_algo_fn auto_algo;
  set_param_fn set_param;
  op_count_fn op_count;
  b2_segment_t seg;

  CHECK(argc == 2);
  lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
  if (!lib) {
    fprintf(stderr, "dlopen: %s\n", dlerror());
    return 1;
  }
  for (i = 0; i < sizeof(symbols) / sizeof(symbols[0]); ++i) {
    if (!dlsym(lib, symbols[i])) {
      fprintf(stderr, "missing symbol %s\n", symbols[i]);
      return 1;
    }
  }
  *(void**)(&version) = dlsym(lib, "b2_version");
  *(void**)(&last_error) = dlsym(lib, "b2_last_error");
  *(void**)(&allreduce) = dlsym(lib, "b2_allreduce");
  *(void**)(&destroy) = dlsym(lib, "b2_comm_destroy");
  CHECK(version() == B2_ABI_VERSION);
  CHECK(allreduce(NULL, NULL, 8, B2_F32_WIRE_BF16, 1.0f, B2_ALGO_AUTO, NULL) == B2_EINVAL);
  CHECK(last_error() != NULL && strlen(last_error()) > 0);
  CHECK(destroy(NULL) == B2_OK);
  *(void**)(&auto_algo) = dlsym(lib, "b2_auto_algo");
  CHECK(auto_algo(8, B2_F32_WIRE_BF16, (size_t)1 << 28, 1) == B2_ALGO_NVLS); /* 1 GiB of fp32 at W=8 with multicast */
  CHECK(auto_algo(8, B2_F32_WIRE_BF16, (size_t)1 << 28, 0) == B2_ALGO_TWOSHOT);
  CHECK(auto_algo(8, B2_F32_WIRE_BF16, 1024, 0) == B2_ALGO_ONESHOT);
  *(void**)(&set_param) = dlsym(lib, "b2_comm_set_param");
  *(void**)(&op_count) = dlsym(lib, "b2_comm_op_count");
  CHECK(set_param(NULL, "op_count", 1) == B2_EINVAL);
  CHECK(op_count(NULL) == 0 && strstr(last_error(), "null communicator") != NULL);
  /* plain-data layout of the one struct that crosses the boundary */
  memset(&seg, 0, sizeof seg);
  CHECK(sizeof seg == sizeof(void*) + 2 * sizeof(uint64_t));
  CHECK(B2_MAX_WORLD == 8 && B2_MAX_SEGMENTS >= 1);
  printf("ok %u symbols abi %d\n", (unsigned)(sizeof(symbols) / sizeof(symbols[0])), version());
  dlclose(lib);
  return 0;
}
