// zk_probe_seed.cu — test-only probe of the seeded expansion (zk_seed.cuh): the 32-byte draw routine with a modulus
// the caller chooses, so that moduli far below 2^256 exercise the rejection branch that the real moduli (2^-32 per
// candidate) essentially never take.
//
// Built like zk_probe.cu: nvcc for sm_90a (libzkprobe_seed.so) and g++ with -DZKA_HOSTSIM (libzkprobe_seed_host.so).
// Never loaded by the product.  Returns 0, -1 for a bad argument, -2 for a CUDA error.
#include "zk_seed.cuh"
#include "zk_launch.cuh"

using namespace zk;

namespace {

struct DrawTask {
  const uint8_t* seeds;     // [count][32]
  const uint64_t* index;    // [count]
  uint32_t domain;
  const uint32_t* mod;      // 8 little-endian limbs
  uint8_t* out;             // [count][32]
  ZK_HD void operator()(int i) const {
    uint32_t key[8], m[8], w[8];
    seed_key(key, seeds + (size_t)i * 32);
    for (int j = 0; j < 8; j++) m[j] = mod[j];
    seed_draw32(w, key, domain, index[i], m);
    st8v(reinterpret_cast<uint32_t*>(out + (size_t)i * 32), w);
  }
};

struct Buf {
  void* p = nullptr;
  explicit Buf(size_t n) : p(dev_alloc(n)) {}
  ~Buf() { dev_free(p); }
  template <class T> T* as() const { return static_cast<T*>(p); }
};

}  // namespace

extern "C" {

// out[i] = the 32 bytes of rnd(mod) on stream(seeds[i], domain, index[i]).  mod >= 2^255 (a candidate passes with
// probability > 1/2, so the loop ends); smaller moduli are refused.
int probe_seed_draw(int count, const uint8_t* seeds, uint32_t domain, const uint64_t* index, const uint32_t* mod, uint8_t* out) {
  if (count < 0 || !(mod[7] & 0x80000000u)) return -1;
  try {
    Buf ds((size_t)count * 32), di((size_t)count * 8), dm(32), dout((size_t)count * 32);
    Stream st;
    copy_h2d(st, ds.p, seeds, (size_t)count * 32);
    copy_h2d(st, di.p, index, (size_t)count * 8);
    copy_h2d(st, dm.p, mod, 32);
    launch(st, count, DrawTask{ds.as<uint8_t>(), di.as<uint64_t>(), domain, dm.as<uint32_t>(), dout.as<uint8_t>()});
    copy_d2h(st, out, dout.p, (size_t)count * 32);
    sync(st);
    return 0;
  } catch (const std::exception&) {
    return -2;
  }
}

}  // extern "C"
