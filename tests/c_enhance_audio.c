/* A C caller of the audio call (fsn_model_enhance_audio): no torch, no FFT library, only the header, the built library and the CUDA
 * runtime.  Used by tests/test_gpu_audio_offline.py.
 *
 *   c_enhance_audio <model file> <wave file> <output file>
 *
 * model file: the fsn_config struct as raw bytes, int32 n, then n records (int32 key length, key bytes, int64 numel, numel float32).
 * wave file: int32 B, int64 L, B int64 lengths, B * L float32 samples.  output file: B * L float32, the enhanced waveforms. */
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "fsnplus_b200.h"

static void need(int ok, const char* what) {
    if (!ok) {
        fprintf(stderr, "c_enhance_audio: %s\n", what);
        exit(1);
    }
}
static void check(int rc, const char* what) {
    if (rc != FSN_OK) {
        fprintf(stderr, "c_enhance_audio: %s failed (%d): %s\n", what, rc, fsn_last_error());
        exit(1);
    }
}

int main(int argc, char** argv) {
    need(argc == 4, "usage: c_enhance_audio <model file> <wave file> <output file>");
    FILE* f = fopen(argv[1], "rb");
    need(f != NULL, "cannot open the model file");
    fsn_config cfg;
    int32_t n = 0;
    need(fread(&cfg, sizeof(cfg), 1, f) == 1 && fread(&n, 4, 1, f) == 1, "short model file");
    fsn_model* m = NULL;
    check(fsn_model_create(&cfg, &m), "fsn_model_create");
    for (int32_t i = 0; i < n; ++i) {
        int32_t klen = 0;
        int64_t numel = 0;
        char key[256];
        need(fread(&klen, 4, 1, f) == 1 && klen > 0 && klen < 256, "bad key length");
        need(fread(key, 1, (size_t)klen, f) == (size_t)klen && fread(&numel, 8, 1, f) == 1, "short parameter record");
        key[klen] = 0;
        float* data = (float*)malloc((size_t)numel * sizeof(float));
        need(data != NULL && fread(data, sizeof(float), (size_t)numel, f) == (size_t)numel, "short parameter data");
        check(fsn_model_set_param(m, key, data, numel), key);
        free(data);
    }
    fclose(f);
    check(fsn_model_finalize(m), "fsn_model_finalize");

    f = fopen(argv[2], "rb");
    need(f != NULL, "cannot open the wave file");
    int32_t B = 0;
    int64_t L = 0;
    need(fread(&B, 4, 1, f) == 1 && fread(&L, 8, 1, f) == 1 && B > 0 && L > 0, "bad wave header");
    int64_t* lengths = (int64_t*)malloc((size_t)B * sizeof(int64_t));
    float* wave = (float*)malloc((size_t)B * (size_t)L * sizeof(float));
    need(lengths && wave, "out of host memory");
    need(fread(lengths, 8, (size_t)B, f) == (size_t)B && fread(wave, sizeof(float), (size_t)B * (size_t)L, f) == (size_t)B * (size_t)L,
         "short wave file");
    fclose(f);

    const size_t bytes = (size_t)B * (size_t)L * sizeof(float);
    float *d_wave = NULL, *d_out = NULL;
    need(cudaMalloc((void**)&d_wave, bytes) == cudaSuccess && cudaMalloc((void**)&d_out, bytes) == cudaSuccess, "cudaMalloc failed");
    need(cudaMemcpy(d_wave, wave, bytes, cudaMemcpyHostToDevice) == cudaSuccess, "cudaMemcpy failed");
    check(fsn_model_enhance_audio(m, d_wave, B, L, lengths, d_out, NULL), "fsn_model_enhance_audio");
    need(cudaMemcpy(wave, d_out, bytes, cudaMemcpyDeviceToHost) == cudaSuccess, "cudaMemcpy failed");

    f = fopen(argv[3], "wb");
    need(f != NULL && fwrite(wave, sizeof(float), (size_t)B * (size_t)L, f) == (size_t)B * (size_t)L, "cannot write the output");
    fclose(f);
    cudaFree(d_wave);
    cudaFree(d_out);
    fsn_model_destroy(m);
    free(wave);
    free(lengths);
    printf("c_enhance_audio: enhanced %d clips\n", B);
    return 0;
}
