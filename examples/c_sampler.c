/*
 * A plain C caller of the drop-in boundary (include/difflinker_b200.h): the reverse-diffusion sampler of
 * EDM.sample_chain (reference src/edm.py:126-235), or of InpaintingEDM.sample_chain (edm.py:549-727) for a model built
 * with centering, without Python and without a noise tensor.
 *
 *   c_sampler [--retries k] <job.bin> <out.bin>
 *
 * job.bin (little endian, written by difflinker_b200/export_job.py from a DDPM and a batch) holds the dl_config (magic
 * DLJOB2: followed by the model's dl_egnn_options -- tanh, mean aggregation), the weights under the reference's state_dict names, the normalised inputs and masks of one batch, the per-step
 * coefficient table of the noise schedule and a Philox (seed, offset) pair; the noise of the T+2 draws (2T+3 for
 * inpainting) is generated inside the kernels (dl_sample_chain_rng) in the order the reference's torch.randn calls would
 * have produced it on this GPU. A seeded job (magic DLJOB3: an int32 flag and, if set, the dl_egnn_options follow the
 * dl_config) holds one uint64 seed per molecule instead of the pair and samples with dl_sample_chain_seeded: each molecule
 * then draws what it would draw sampled alone, so any molecule can be replayed from its seed.
 * out.bin: int32 status, uint64 philox offset consumed (0 for a seeded job), the (keep_frames, B, N, 3+F) chain,
 * B NaN flags. `--retries k` (seeded jobs only) samples with dl_sample_chain_retry instead: up to k rounds resample
 * the molecules that diverged with new seeds (dl_retry_seed), and out.bin goes on with the B uint64 seeds that produced the
 * rows and the B int32 attempts (0 = the first draw); only rows that still fail keep their flags.
 *
 * Build: gcc -std=c99 -O2 examples/c_sampler.c -Iinclude -I/usr/local/cuda/include -Ldifflinker_b200 -ldifflinker_b200 \
 *            -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,$PWD/difflinker_b200 -o c_sampler
 */
#include <cuda_runtime_api.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "difflinker_b200.h"

static void die(const char* what) {
  fprintf(stderr, "c_sampler: %s (%s)\n", what, dl_last_error());
  exit(2);
}
static void rd(FILE* f, void* p, size_t n) {
  if (n && fread(p, 1, n, f) != n) { fprintf(stderr, "c_sampler: short read\n"); exit(2); }
}
static void* rd_alloc(FILE* f, size_t n) {
  void* p = malloc(n ? n : 1);
  if (!p) { fprintf(stderr, "c_sampler: out of memory\n"); exit(2); }
  rd(f, p, n);
  return p;
}
static void* to_device(const void* host, size_t n) {
  void* d = NULL;
  if (cudaMalloc(&d, n ? n : 1) != cudaSuccess || cudaMemcpy(d, host, n, cudaMemcpyHostToDevice) != cudaSuccess) {
    fprintf(stderr, "c_sampler: device copy of %zu bytes failed\n", n);
    exit(2);
  }
  return d;
}

int main(int argc, char** argv) {
  int32_t retries = -1;                          /* -1: no recovery rounds (dl_sample_chain_seeded) */
  if (argc == 5 && strcmp(argv[1], "--retries") == 0) {
    char* end = NULL;
    const long k = strtol(argv[2], &end, 10);
    if (*argv[2] == 0 || *end != 0 || k < 0 || k > 1000000) { fprintf(stderr, "c_sampler: bad --retries %s\n", argv[2]); return 2; }
    retries = (int32_t)k;
    argv += 2;
    argc -= 2;
  }
  if (argc != 3) { fprintf(stderr, "usage: %s [--retries k] job.bin out.bin\n", argv[0]); return 2; }
  FILE* f = fopen(argv[1], "rb");
  if (!f) { perror(argv[1]); return 2; }
  char magic[8];
  rd(f, magic, 8);
  const int seeded = memcmp(magic, "DLJOB3\0\0", 8) == 0;
  int32_t with_opts = memcmp(magic, "DLJOB2\0\0", 8) == 0;
  if (!seeded && !with_opts && memcmp(magic, "DLJOB1\0\0", 8) != 0) { fprintf(stderr, "c_sampler: not a job file\n"); return 2; }
  if (retries >= 0 && !seeded) { fprintf(stderr, "c_sampler: --retries needs a seeded (DLJOB3) job\n"); return 2; }

  dl_config cfg;
  rd(f, &cfg, sizeof cfg);                       /* 11 int32 + 2 float, no padding (checked by the exporter) */
  if (seeded) rd(f, &with_opts, 4);
  dl_egnn_options opts;
  if (with_opts) rd(f, &opts, sizeof opts);      /* 3 int32 + 1 float */
  dl_engine* e = NULL;
  if (dl_create_ex(&cfg, with_opts ? &opts : NULL, &e) < 0) die("dl_create_ex");

  int32_t n_weights;
  rd(f, &n_weights, 4);
  for (int32_t i = 0; i < n_weights; ++i) {
    int32_t len; int64_t numel; char name[256];
    rd(f, &len, 4);
    if (len <= 0 || len >= (int32_t)sizeof name) { fprintf(stderr, "c_sampler: bad weight name\n"); return 2; }
    rd(f, name, (size_t)len);
    name[len] = 0;
    rd(f, &numel, 8);
    float* w = (float*)rd_alloc(f, (size_t)numel * 4);
    if (dl_set_weight(e, name, w, numel) < 0) die(name);
    free(w);
  }
  if (dl_finalize_weights(e) < 0) die("dl_finalize_weights");

  int32_t dims[6];                               /* B, N, T, keep_frames, xd = 3 + F, C */
  uint64_t rng[2] = {0, 0};                      /* philox seed, offset */
  float norm[3];
  rd(f, dims, sizeof dims);
  const int32_t B = dims[0], N = dims[1], T = dims[2], keep = dims[3], xd = dims[4], C = dims[5];
  const size_t n = (size_t)B * N;
  uint64_t* seeds = seeded ? (uint64_t*)rd_alloc(f, (size_t)B * 8) : NULL;   /* seeded job: one seed per molecule */
  if (!seeded) rd(f, rng, sizeof rng);
  rd(f, norm, sizeof norm);
  dl_step_coef* coef = (dl_step_coef*)rd_alloc(f, (size_t)(T + 1) * sizeof(dl_step_coef));   /* host table, as the ABI asks */
  float* xh = (float*)rd_alloc(f, n * xd * 4);
  int8_t* node_mask = (int8_t*)rd_alloc(f, n);
  float* fragment_mask = (float*)rd_alloc(f, n * 4);
  float* linker_mask = (float*)rd_alloc(f, n * 4);
  int32_t has_em, has_ctx;
  rd(f, &has_em, 4);
  int8_t* edge_mask = has_em ? (int8_t*)rd_alloc(f, n * N) : NULL;
  rd(f, &has_ctx, 4);
  float* context = has_ctx ? (float*)rd_alloc(f, n * C * 4) : NULL;
  fclose(f);

  if (cudaSetDevice(cfg.device) != cudaSuccess) { fprintf(stderr, "c_sampler: no CUDA device %d\n", cfg.device); return 2; }
  float* d_xh = (float*)to_device(xh, n * xd * 4);
  int8_t* d_nm = (int8_t*)to_device(node_mask, n);
  float* d_fm = (float*)to_device(fragment_mask, n * 4);
  float* d_lm = (float*)to_device(linker_mask, n * 4);
  int8_t* d_em = has_em ? (int8_t*)to_device(edge_mask, n * N) : NULL;
  float* d_ctx = has_ctx ? (float*)to_device(context, n * C * 4) : NULL;
  uint64_t* d_seeds = seeded ? (uint64_t*)to_device(seeds, (size_t)B * 8) : NULL;
  float* d_chain = NULL;
  int32_t* d_flags = NULL;
  uint64_t* d_used = NULL;
  int32_t* d_attempts = NULL;
  const size_t chain_bytes = (size_t)keep * n * xd * 4;
  if (cudaMalloc((void**)&d_chain, chain_bytes) != cudaSuccess || cudaMalloc((void**)&d_flags, (size_t)B * 4) != cudaSuccess ||
      cudaMalloc((void**)&d_used, (size_t)B * 8) != cudaSuccess || cudaMalloc((void**)&d_attempts, (size_t)B * 4) != cudaSuccess) {
    fprintf(stderr, "c_sampler: cudaMalloc failed\n");
    return 2;
  }
  cudaStream_t stream;
  if (cudaStreamCreate(&stream) != cudaSuccess) { fprintf(stderr, "c_sampler: cudaStreamCreate failed\n"); return 2; }

  uint64_t consumed = 0;
  /* inpainting models are the ones built with centering (lightning.py:99); the engine refuses any other pairing */
  const int32_t sampler = cfg.centering ? DL_SAMPLER_INPAINT : DL_SAMPLER_LINKER;
  dl_status st;
  if (retries >= 0)   /* blocks until its rounds are done */
    st = dl_sample_chain_retry(e, sampler, B, N, T, keep, d_xh, d_nm, d_fm, d_lm, d_em, d_ctx, d_seeds, coef, norm, d_chain,
                               d_flags, retries, d_used, d_attempts, NULL, NULL, NULL, NULL, stream);
  else if (seeded)
    st = dl_sample_chain_seeded(e, sampler, B, N, T, keep, d_xh, d_nm, d_fm, d_lm, d_em, d_ctx, d_seeds, coef, norm, d_chain,
                                d_flags, stream);
  else
    st = dl_sample_chain_rng(e, sampler, B, N, T, keep, d_xh, d_nm, d_fm, d_lm, d_em, d_ctx, rng[0], rng[1], &consumed, coef,
                             norm, d_chain, d_flags, stream);
  if (st < 0) die(retries >= 0 ? "dl_sample_chain_retry" : seeded ? "dl_sample_chain_seeded" : "dl_sample_chain_rng");
  if (cudaStreamSynchronize(stream) != cudaSuccess) { fprintf(stderr, "c_sampler: the sampler's stream failed\n"); return 2; }

  float* chain = (float*)malloc(chain_bytes);
  int32_t* flags = (int32_t*)malloc((size_t)B * 4);
  cudaMemcpy(chain, d_chain, chain_bytes, cudaMemcpyDeviceToHost);
  cudaMemcpy(flags, d_flags, (size_t)B * 4, cudaMemcpyDeviceToHost);
  FILE* o = fopen(argv[2], "wb");
  if (!o) { perror(argv[2]); return 2; }
  const int32_t status = (int32_t)st;
  fwrite(&status, 4, 1, o);
  fwrite(&consumed, 8, 1, o);
  fwrite(chain, 1, chain_bytes, o);
  fwrite(flags, 4, (size_t)B, o);
  if (retries >= 0) {
    uint64_t* used = (uint64_t*)malloc((size_t)B * 8);
    int32_t* attempts = (int32_t*)malloc((size_t)B * 4);
    cudaMemcpy(used, d_used, (size_t)B * 8, cudaMemcpyDeviceToHost);
    cudaMemcpy(attempts, d_attempts, (size_t)B * 4, cudaMemcpyDeviceToHost);
    fwrite(used, 8, (size_t)B, o);
    fwrite(attempts, 4, (size_t)B, o);
    printf("c_sampler: %d recovery round(s) allowed, %.2f ms of retry rounds on the device\n", retries, dl_last_retry_ms(e));
    free(used);
    free(attempts);
  }
  fclose(o);
  printf("c_sampler: %d molecules x %d atoms, T=%d: %.2f ms on the device, %lld kernels, philox offset +%llu\n", B, N, T,
         dl_last_elapsed_ms(e), (long long)dl_launch_count(e), (unsigned long long)consumed);
  dl_destroy(e);
  return 0;
}
