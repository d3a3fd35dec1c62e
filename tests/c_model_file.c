/* A C caller of a model file: fsn_model_load gives a ready handle, fsn_model_enhance_audio enhances a batch of clips.  No torch, no
 * parameter plumbing: only the header, the built library and the CUDA runtime.  Used by tests/test_gpu_model_file.py.
 *
 *   c_model_file <model file> <wave file> <output file>
 *
 * wave file: int32 B, int64 L, B int64 lengths, B * L float32 samples.  output file: B * L float32, the enhanced waveforms.  Prints the
 * handle's weights_id. */
#include <stdio.h>
#include <stdlib.h>

#include <cuda_runtime.h>

#include "fsnplus_b200.h"

static void need(int ok, const char* what) {
    if (!ok) {
        fprintf(stderr, "c_model_file: %s\n", what);
        exit(1);
    }
}
static void check(int rc, const char* what) {
    if (rc != FSN_OK) {
        fprintf(stderr, "c_model_file: %s failed (%d): %s\n", what, rc, fsn_last_error());
        exit(1);
    }
}

int main(int argc, char** argv) {
    need(argc == 4, "usage: c_model_file <model file> <wave file> <output file>");
    fsn_model* m = NULL;
    check(fsn_model_load(argv[1], &m), "fsn_model_load");

    FILE* f = fopen(argv[2], "rb");
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
    need(fclose(f) == 0, "cannot write the output");
    printf("c_model_file: weights_id %016llx, enhanced %d clips\n", (unsigned long long)fsn_model_weights_id(m), B);
    cudaFree(d_wave);
    cudaFree(d_out);
    fsn_model_destroy(m);
    free(wave);
    free(lengths);
    return 0;
}
