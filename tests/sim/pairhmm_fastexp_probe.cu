// Probe of tests/test_pairhmm.py: FastExp as the pair-HMM kernels inline it must compile to separate DMUL / DADD
// (bit-identical to the host's), while a plain a * b + c beside it shows that the compiler would contract one.
#include "../../rust_bio_b200/csrc/b2a_pairhmm.cuh"

__global__ void fastexp_probe(const double* in, double* out) { out[threadIdx.x] = b2a::ph_fastexp(in[threadIdx.x]); }
__global__ void contract_probe(const double* in, double* out) { out[threadIdx.x] = in[threadIdx.x] * 3.0 + 1.0; }
