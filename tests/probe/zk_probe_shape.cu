// zk_probe_shape.cu — test-only probe of the fixed-base table shape (FbShape, zk_ops.cuh): the layout helpers and the
// signed-digit recoding of scalars on a table whose windows are w or w + 1 bits wide.
//
// Built like zk_probe.cu: nvcc for sm_90a (libzkprobe_shape.so) and g++ with -DZKA_HOSTSIM (libzkprobe_shape_host.so).
// Never loaded by the product.  Returns 0, -1 for a bad argument, -2 for a CUDA error.
#include "zk_ops.cuh"
#include "zk_launch.cuh"

using namespace zk;

namespace {

enum : int { SHAPE_ROW = 132 };   // digits of one scalar, the carry out of the top window at [131]

struct ShapeDigitTask {
  FbShape sh;
  const uint32_t* scalars;   // [count][8]
  int32_t* out;              // [count][SHAPE_ROW]
  ZK_HD void operator()(int i) const {
    const uint32_t* k = scalars + (size_t)i * 8;
    int32_t* o = out + (size_t)i * SHAPE_ROW;
    uint32_t carry = 0;
    for (int j = 0; j < sh.nwin; j++) {
      bool neg;
      const uint32_t d = signed_digit(k, j, sh, carry, neg);
      o[j] = neg ? -(int32_t)d : (int32_t)d;
    }
    o[SHAPE_ROW - 1] = (int32_t)carry;
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

// the shape for `nwin` lookups (uniform_w = 0) or the uniform shape of uniform_w bits: head = {w, nwin, n_lo, bits},
// layout[j] = {width, bit position, entries, entry offset} of window j, layout[nwin] = {0, bits, 0, total entries}
int probe_shape(int nwin, int uniform_w, int64_t* head, int64_t* layout) {
  if (uniform_w ? (uniform_w < 2 || uniform_w > 24) : (nwin < 11 || nwin > 128)) return -1;
  const FbShape sh = uniform_w ? fb_uniform(uniform_w) : fb_lookups(nwin);
  head[0] = sh.w; head[1] = sh.nwin; head[2] = sh.n_lo; head[3] = sh.bits();
  for (int j = 0; j <= sh.nwin; j++) {
    int64_t* l = layout + 4 * j;
    l[0] = j < sh.nwin ? sh.width(j) : 0;
    l[1] = sh.bitpos(j);
    l[2] = j < sh.nwin ? (int64_t)sh.entries(j) : 0;
    l[3] = (int64_t)sh.offset(j);
  }
  return 0;
}

// signed digits of each 8-limb scalar on that shape: out[i] = nwin digits, the carry out of the top window at [131]
int probe_shape_digits(int nwin, int uniform_w, int count, const uint32_t* scalars, int32_t* out) {
  if (count < 0 || (uniform_w ? (uniform_w < 2 || uniform_w > 24) : (nwin < 11 || nwin > 128))) return -1;
  const FbShape sh = uniform_w ? fb_uniform(uniform_w) : fb_lookups(nwin);
  try {
    Buf ds((size_t)count * 32), dout((size_t)count * SHAPE_ROW * 4);
    Stream st;
    copy_h2d(st, ds.p, scalars, (size_t)count * 32);
    dev_memset(st, dout.p, 0, (size_t)count * SHAPE_ROW * 4);
    launch(st, count, ShapeDigitTask{sh, ds.as<uint32_t>(), dout.as<int32_t>()});
    copy_d2h(st, out, dout.p, (size_t)count * SHAPE_ROW * 4);
    sync(st);
    return 0;
  } catch (const std::exception&) {
    return -2;
  }
}

}  // extern "C"
