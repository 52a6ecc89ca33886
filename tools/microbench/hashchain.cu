// hashchain.cu — the hash_chain kernel against hash_generic, the fully serial kernel that hashes every block as one
// XXH64 message (no pre-state split): bit-exact chains and block counts on ragged, unaligned and truncated prompts
// (block sizes 32, 64, 96, 128, 160 and 256, odd batch sizes, every tile shape), then CUDA-event times of hash_chain at the cfg 3
// shape (16 384 requests x 4 096-token prompts, 64-byte blocks, 256 blocks), the cfg 2 shape (4 096 requests x
// 2 048-token prompts) and the cfg 3 shape at 96- and 160-byte blocks.  Prints one line per case.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I fusioninfer_b200/csrc -o tools/microbench/hashchain tools/microbench/hashchain.cu
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <vector>

#include "hash_kernels.cu"

#define CK(x)                                                                              \
  do {                                                                                     \
    cudaError_t e_ = (x);                                                                  \
    if (e_ != cudaSuccess) {                                                               \
      std::fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); \
      std::exit(1);                                                                        \
    }                                                                                      \
  } while (0)

static int g_sms = 132;

struct Batch {
  uint32_t R, B, M, MP;
  uint8_t* prompts;
  uint64_t *offsets, *h0, *chain_a, *chain_b;
  uint32_t *nb_a, *nb_b;
};

// ragged: lengths uniform in [0, (M + 4) * B - 1] and random byte gaps between prompts (unaligned starts)
static Batch make_batch(uint32_t R, uint32_t B, uint32_t M, bool ragged, uint64_t seed) {
  Batch b{R, B, M, (M + 7) & ~7u};
  std::mt19937_64 rng(seed);
  std::vector<uint64_t> off(R + 1);
  uint64_t at = 0;
  for (uint32_t r = 0; r < R; ++r) {
    if (ragged) at += rng() % 24;
    off[r] = at;
    at += ragged ? rng() % ((uint64_t)(M + 4) * B) : (uint64_t)M * B;
  }
  off[R] = at;
  std::vector<uint8_t> bytes(at + 64);
  for (auto& x : bytes) x = (uint8_t)rng();
  std::vector<uint64_t> h0(R);
  for (auto& x : h0) x = rng();
  CK(cudaMalloc(&b.prompts, bytes.size()));
  CK(cudaMalloc(&b.offsets, (R + 1) * sizeof(uint64_t)));
  CK(cudaMalloc(&b.h0, R * sizeof(uint64_t)));
  CK(cudaMalloc(&b.chain_a, (size_t)R * b.MP * sizeof(uint64_t)));
  CK(cudaMalloc(&b.chain_b, (size_t)R * b.MP * sizeof(uint64_t)));
  CK(cudaMalloc(&b.nb_a, R * sizeof(uint32_t)));
  CK(cudaMalloc(&b.nb_b, R * sizeof(uint32_t)));
  CK(cudaMemcpy(b.prompts, bytes.data(), bytes.size(), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(b.offsets, off.data(), off.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(b.h0, h0.data(), h0.size() * sizeof(uint64_t), cudaMemcpyHostToDevice));
  CK(cudaMemset(b.chain_a, 0xA5, (size_t)R * b.MP * sizeof(uint64_t)));
  CK(cudaMemset(b.chain_b, 0x5A, (size_t)R * b.MP * sizeof(uint64_t)));
  return b;
}
static void free_batch(Batch& b) {
  cudaFree(b.prompts), cudaFree(b.offsets), cudaFree(b.h0);
  cudaFree(b.chain_a), cudaFree(b.chain_b), cudaFree(b.nb_a), cudaFree(b.nb_b);
}
static void run_generic(Batch& b) {
  CK(fi::launch_hash_generic(b.prompts, b.offsets, b.h0, b.R, b.B, b.M, b.MP, b.chain_a, b.nb_a, 0));
}
// walk = 0: the shape launch_hash_chain picks for the batch
static void run_chain(Batch& b, uint32_t walk = 0, uint32_t warps = 0) {
  if (walk)
    CK(fi::launch_hash_chain_shape(walk, warps, b.prompts, b.offsets, b.h0, b.R, b.B, b.M, b.MP, b.chain_b, b.nb_b, 0));
  else
    CK(fi::launch_hash_chain(b.prompts, b.offsets, b.h0, b.R, b.B, b.M, b.MP, b.chain_b, b.nb_b, g_sms, 0));
}
static bool same(const Batch& b) {
  std::vector<uint64_t> ca((size_t)b.R * b.MP), cb(ca.size());
  std::vector<uint32_t> na(b.R), nb(b.R);
  CK(cudaMemcpy(ca.data(), b.chain_a, ca.size() * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(cb.data(), b.chain_b, cb.size() * 8, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(na.data(), b.nb_a, na.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(nb.data(), b.nb_b, nb.size() * 4, cudaMemcpyDeviceToHost));
  return ca == cb && na == nb;
}

// hash_chain alone, 3 x 50 launches; the outputs of the last one against hash_generic
static bool time_shape(const char* name, uint32_t R, uint32_t B, uint32_t M, uint32_t walk = 0, uint32_t warps = 0) {
  Batch b = make_batch(R, B, M, false, 3);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0));
  CK(cudaEventCreate(&e1));
  for (int w = 0; w < 5; ++w) run_chain(b, walk, warps);
  CK(cudaDeviceSynchronize());
  const int iters = 50;
  for (int rep = 0; rep < 3; ++rep) {
    float ms = 0;
    for (int it = 0; it < iters; ++it) {
      float t;
      CK(cudaEventRecord(e0));
      run_chain(b, walk, warps);
      CK(cudaEventRecord(e1));
      CK(cudaEventSynchronize(e1));
      CK(cudaEventElapsedTime(&t, e0, e1));
      ms += t;
    }
    std::printf("%s (B=%u, %u blocks) rep %d: hash_chain %.1f us\n", name, B, M, rep, 1e3 * ms / iters);
  }
  run_generic(b);
  CK(cudaDeviceSynchronize());
  const bool ok = same(b);
  std::printf("%s outputs %s\n", name, ok ? "identical" : "DIFFER");
  CK(cudaEventDestroy(e0));
  CK(cudaEventDestroy(e1));
  free_batch(b);
  return ok;
}

int main() {
  int fails = 0;
  CK(cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0));
  // correctness: compiled-in (32, 64, 128) and run-time (96, 160, 256) stripe counts, ragged + unaligned +
  // truncated, batch sizes with a partial last tile
  const uint32_t Rs[] = {1, 31, 129, 1000};
  const uint32_t Bs[] = {32, 64, 96, 128, 160, 256};
  const uint32_t Ms[] = {5, 100, 256};
  for (uint32_t R : Rs)
    for (uint32_t B : Bs)
      for (uint32_t M : Ms)
        for (int ragged = 0; ragged < 2; ++ragged) {
          Batch b = make_batch(R, B, M, ragged, R * 7919ull + B * 31 + M + ragged);
          run_generic(b);
          const uint32_t shapes[3][2] = {{1, 32}, {2, 32}, {2, 16}};  // whole-SM WALK = 1, 2 and the half-SM tile
          for (auto& sh : shapes) {
            CK(cudaMemset(b.chain_b, 0x5A, (size_t)b.R * b.MP * sizeof(uint64_t)));
            run_chain(b, sh[0], sh[1]);
            CK(cudaDeviceSynchronize());
            if (!same(b)) {
              ++fails;
              std::printf("MISMATCH R=%u B=%u M=%u ragged=%d walk=%u warps=%u\n", R, B, M, ragged, sh[0], sh[1]);
            }
          }
          free_batch(b);
        }
  std::printf("correctness: %d mismatching case(s) of %zu\n", fails, sizeof(Rs) / 4 * sizeof(Bs) / 4 * sizeof(Ms) / 4 * 2 * 3);

  // timing at cfg 3 (16 384 x 256 blocks: half-SM tiles of 64 requests, against whole-SM tiles of 64), cfg 2
  // (4 096 x 128 blocks: 32 per whole-SM CTA, against half-SM tiles), and the cfg 3 prompts (16 KiB each) cut into
  // 96- and 160-byte blocks
  bool ok = time_shape("cfg3", 16384, 64, 256);
  ok = time_shape("cfg3 whole-SM WALK=2", 16384, 64, 256, 2, 32) && ok;
  ok = time_shape("cfg2", 4096, 64, 128) && ok;
  ok = time_shape("cfg2 half-SM", 4096, 64, 128, 2, 16) && ok;
  ok = time_shape("cfg3-96B", 16384, 96, 16384 / 96) && ok;
  ok = time_shape("cfg3-160B", 16384, 160, 16384 / 160) && ok;
  return (fails || !ok) ? 1 : 0;
}
