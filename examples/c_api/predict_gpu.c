/*
 * Serve a saved checkpoint on GPU 0 through the flat C ABI only — no Python, no PyTorch in the process: the serving half of train_cnn.c
 * with dev_type 2, so the planned predictor runs its graph as sm_90a kernels.
 *   GXPredCreate (dev_type 2)   upload the parameters, plan the arena      GXPredSetInput / GXPredForward / GXPredGetOutput   one batch
 *
 *   gcc -O2 -I geomx_b200/include examples/c_api/predict_gpu.c -L geomx_b200/lib -lgeomx_capi -Wl,-rpath,$PWD/geomx_b200/lib -o predict_gpu
 *   ./predict_gpu net-symbol.json net-0001.params input.f32 N C H W > output.txt
 *
 * input.f32 holds N*C*H*W float32 values (the "data" input, NCHW); the program prints every value of output 0, one per line.
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include "geomx/c_api.h"

#define CK(x)                                                                           \
  do {                                                                                  \
    if ((x) != 0) {                                                                     \
      fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, GXRTGetLastError());    \
      return 1;                                                                         \
    }                                                                                   \
  } while (0)

static char* read_file(const char* path, long* size) {
  FILE* f = fopen(path, "rb");
  char* buf;
  if (f == NULL) return NULL;
  fseek(f, 0, SEEK_END); *size = ftell(f); fseek(f, 0, SEEK_SET);
  buf = (char*)calloc((size_t)*size + 1, 1);
  if (buf != NULL && fread(buf, 1, (size_t)*size, f) != (size_t)*size) { free(buf); buf = NULL; }
  fclose(f);
  return buf;
}

int main(int argc, char** argv) {
  long jsz = 0, psz = 0, xsz = 0;
  char *json, *params, *input;
  uint32_t dims[4], ind[2] = {0, 4}, *oshape, ondim, i, n = 1;
  const char* keys[1] = {"data"};
  PredictorHandle pred;
  float* out;
  int engine;
  if (argc < 8) {
    fprintf(stderr, "usage: %s symbol.json file.params input.f32 N C H W\n", argv[0]);
    return 2;
  }
  for (i = 0; i < 4; ++i) dims[i] = (uint32_t)atoi(argv[4 + i]);
  json = read_file(argv[1], &jsz); params = read_file(argv[2], &psz); input = read_file(argv[3], &xsz);
  if (json == NULL || params == NULL || input == NULL) { fprintf(stderr, "cannot read the inputs\n"); return 2; }
  if ((uint64_t)xsz != (uint64_t)dims[0] * dims[1] * dims[2] * dims[3] * sizeof(float)) { fprintf(stderr, "input.f32 does not hold N*C*H*W floats\n"); return 2; }

  CK(GXPredCreate(json, params, (int)psz, 2, 0, 1, keys, ind, dims, &pred));
  CK(GXPredGetEngine(pred, &engine));
  CK(GXPredSetInput(pred, "data", (const float*)input, dims[0] * dims[1] * dims[2] * dims[3]));
  CK(GXPredForward(pred));
  CK(GXPredGetOutputShape(pred, 0, &oshape, &ondim));
  for (i = 0; i < ondim; ++i) n *= oshape[i];
  out = (float*)malloc(n * sizeof(float));
  CK(GXPredGetOutput(pred, 0, out, n));
  fprintf(stderr, "engine %d, %u output values\n", engine, n);
  for (i = 0; i < n; ++i) printf("%.9g\n", out[i]);
  CK(GXPredFree(pred));
  free(out); free(json); free(params); free(input);
  return 0;
}
