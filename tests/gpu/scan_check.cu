// scan_check.cu -- runs the engine's single-pass scans (samtools_b200/csrc/scan.cuh, k_scan) on files of 32-bit inputs, one
// instantiation per stage that launches it, so that tests/test_gpu_scan.py can compare them with numpy.
//   scan_check KIND IN OUT [KIND IN OUT ...]
//   KIND  max8      inclusive max, int32 -> int32, 8 items per thread       (prefix max of read ends)
//         sum4      inclusive sum mod 2^32, int32 -> int32, 4 per thread    (coverage difference array)
//         sum1_u64  exclusive sum + total, uint32 -> uint64, 1 per thread   (tile offsets, entry and GL offsets)
//         sum1_i32  exclusive sum + total, uint32 -> int32, 1 per thread    (far-reaching list offsets)
// OUT gets n outputs (inclusive) or n + 1 (exclusive: the total last).
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../samtools_b200/csrc/scan.cuh"

#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { \
    fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); exit(1); } } while (0)

template <class Op, int IPT, bool INCL, class In, class Out>
static void run(const char *fin, const char *fout)
{
    FILE *f = fopen(fin, "rb");
    if (!f) { fprintf(stderr, "cannot open %s\n", fin); exit(1); }
    std::vector<In> h;
    In x;
    while (fread(&x, sizeof x, 1, f) == 1) h.push_back(x);
    fclose(f);
    const int32_t n = (int32_t)h.size(), n_out = n + (INCL ? 0 : 1);
    const int nb = (n + SCAN_T * IPT - 1) / (SCAN_T * IPT);
    In *d_in; Out *d_out; uint64_t *d_st;
    CK(cudaMalloc(&d_in, h.size() * sizeof(In) + 1)); CK(cudaMalloc(&d_out, (size_t)n_out * sizeof(Out)));
    CK(cudaMalloc(&d_st, ((size_t)nb + 1) * 8));
    CK(cudaMemcpy(d_in, h.data(), h.size() * sizeof(In), cudaMemcpyHostToDevice));
    CK(cudaMemset(d_st, 0, ((size_t)nb + 1) * 8));                // the ticket, then one status word per block
    k_scan<Op, IPT, INCL><<<nb, SCAN_T>>>(d_in, d_out, n, d_st + 1, (uint32_t *)d_st);
    CK(cudaGetLastError());
    std::vector<Out> o((size_t)n_out);
    CK(cudaMemcpy(o.data(), d_out, o.size() * sizeof(Out), cudaMemcpyDeviceToHost));
    CK(cudaFree(d_in)); CK(cudaFree(d_out)); CK(cudaFree(d_st));
    f = fopen(fout, "wb");
    if (!f || fwrite(o.data(), sizeof(Out), o.size(), f) != o.size() || fclose(f)) { fprintf(stderr, "cannot write %s\n", fout); exit(1); }
}

int main(int argc, char **argv)
{
    if (argc < 4 || (argc - 1) % 3) { fprintf(stderr, "usage: scan_check KIND IN OUT [KIND IN OUT ...]\n"); return 2; }
    for (int a = 1; a < argc; a += 3) {
        const char *k = argv[a];
        if (!strcmp(k, "max8")) run<ScanMax, 8, true, int32_t, int32_t>(argv[a + 1], argv[a + 2]);
        else if (!strcmp(k, "sum4")) run<ScanSum, 4, true, int32_t, int32_t>(argv[a + 1], argv[a + 2]);
        else if (!strcmp(k, "sum1_u64")) run<ScanSum, 1, false, uint32_t, uint64_t>(argv[a + 1], argv[a + 2]);
        else if (!strcmp(k, "sum1_i32")) run<ScanSum, 1, false, uint32_t, int32_t>(argv[a + 1], argv[a + 2]);
        else { fprintf(stderr, "unknown kind %s\n", k); return 2; }
    }
    return 0;
}
