// The device hashes behind the library's open-addressed tables, evaluated on the GPU for a list of inputs, so that
// tests/hash_rules.py's restatements (and every collision the tests build from them) are checked value for value.
//   hash_check <in> <out>: <in> holds HcIn records, <out> gets one uint64 per record:
//   kind 0 key_hash(key)            kind 1 key_owner(key, a)        kind 2 join_hash(a, b)
//   kind 3 st_hash(a, b, c, d)      kind 4 st_cand_hash(key, span a, per span)   kind 5 la_hash(key, len)
//   kind 6 st_turn_slot(a, b) at c slots                             kind 7 st_view_slot(a, b, c) at d slots
// nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a
#include <cstdio>
#include <vector>

#include "../distributed_crawler_b200/csrc/local_appends.cuh"
#include "../distributed_crawler_b200/csrc/state.cuh"

using namespace tgi;

struct HcIn {
  uint32_t kind, len;
  uint64_t a, b, c, d;
  uint8_t key[32];
};

__global__ void hash_check_kernel(const HcIn* in, uint64_t n, uint64_t* out) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const HcIn& r = in[i];
  const Key32 k = load_key(r.key);
  uint64_t v = 0;
  switch (r.kind) {
    case 0: v = key_hash(k); break;
    case 1: v = key_owner(k, (uint32_t)r.a); break;
    case 2: v = join_hash((long long)r.a, (long long)r.b); break;
    case 3: v = st_hash((uint32_t)r.a, (uint32_t)r.b, (long long)r.c, (long long)r.d); break;
    case 4: v = st_cand_hash(k, (uint32_t)r.a, true); break;
    case 5: v = la_hash(r.key, r.len); break;
    case 6: {
      StTurn t{};
      t.bmask = r.c - 1;
      v = st_turn_slot(t, (uint32_t)r.a, (long long)r.b);
      break;
    }
    case 7: {
      StView w{};
      w.vmask = r.d - 1;
      v = st_view_slot(w, (uint32_t)r.a, (long long)r.b, (long long)r.c);
      break;
    }
    default: v = ~0ull;
  }
  out[i] = v;
}

int main(int argc, char** argv) {
  if (argc != 3) {
    std::fprintf(stderr, "usage: hash_check <in> <out>\n");
    return 2;
  }
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 2;
  std::vector<HcIn> in;
  HcIn r;
  while (std::fread(&r, sizeof r, 1, f) == 1) in.push_back(r);
  std::fclose(f);
  const uint64_t n = in.size();
  HcIn* d_in = nullptr;
  uint64_t* d_out = nullptr;
  std::vector<uint64_t> out(n);
  if (cudaMalloc(&d_in, n * sizeof(HcIn) + 1) || cudaMalloc(&d_out, n * 8 + 8) ||
      cudaMemcpy(d_in, in.data(), n * sizeof(HcIn), cudaMemcpyHostToDevice)) {
    std::fprintf(stderr, "cuda: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  if (n) hash_check_kernel<<<(unsigned)((n + 255) / 256), 256>>>(d_in, n, d_out);
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess || cudaMemcpy(out.data(), d_out, n * 8, cudaMemcpyDeviceToHost)) {
    std::fprintf(stderr, "cuda: %s\n", cudaGetErrorString(e));
    return 1;
  }
  f = std::fopen(argv[2], "wb");
  if (!f || std::fwrite(out.data(), 8, n, f) != n) return 2;
  std::fclose(f);
  std::printf("ok: %llu hashes\n", (unsigned long long)n);
  return 0;
}
