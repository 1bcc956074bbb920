// zkattest_napi.cc — node-addon-api shim over the C ABI (include/zkattest.h).
// NOT compiled in this image (no node / node-addon-api headers; SURVEY.md F7).  Build where node >= 24 exists:
//   npm i node-addon-api && npx node-gyp configure build       (binding.gyp next to this file)
//
// Exports (used by zkpAttestListGpu.ts):
//   paramsGenerate(rnd64) -> {hNist, hProof}                       zka_params_generate
//   paramsCreate(hNist, hProof, secLevel) -> Params                zka_params_create
//   paramsDestroy(params)                                          zka_params_destroy
//   keyToInt(raw65 x count) -> Promise<Uint8Array(32 x count)>     zka_key_to_int
//   proveBatch(params, msgHash, sig, pk, which, ring, tape, secLevel) -> Promise<{proofs, stride, lens}>
//   verifyBatch(params, msgHash, ring, proofs, lens, stride, tape, secLevel) -> Promise<{ok}>
// The heavy calls are Napi::AsyncWorkers so the TypeScript functions keep returning Promises (the reference is
// async only because of WebCrypto, src/zkpAttestList.ts:104,147).  A zka_ctx runs ONE call at a time (it fans a
// call out over its own lanes internally), and libuv runs workers on a thread pool: every use of the context is
// serialised by g_mu.  status[i] != 0 rejects the promise with the reference's Error message.
#include <napi.h>

#include <mutex>
#include <string>
#include <vector>

#include "zkattest.h"

namespace {

zka_ctx* g_ctx = nullptr;
std::mutex g_mu;

const char* status_message(int s) {
  switch (s) {
    case ZKA_ERR_INVALID_PK: return "invalid public key";          // zkpAttestList.ts:117
    case ZKA_ERR_T_INFINITY: return "T[i] is at infinity";         // exp.ts:151
    case ZKA_ERR_T1_INFINITY: return "T1 is at infinity";          // exp.ts:193
    case ZKA_ERR_POINTS_DONT_ADD: return "Points don't add up!";   // pointAdd.ts:105
    case ZKA_ERR_TAPE_RANGE: return "zkattest: randomness draw out of range";
    case ZKA_ERR_BAD_INDEX: return "zkattest: index outside the ring";
    case ZKA_ERR_IDENTITY_ENC: return "zkattest: identity point in a proof slot";
    case ZKA_ERR_R_INFINITY: return "R is at infinity";            // zkpAttestList.ts:159
    case ZKA_ERR_MALFORMED: return "error deserializing Point";    // weier.ts:87
    case ZKA_ERR_PARAMS_NOT_FOUND: return "params not found";      // exp.ts:270
    case ZKA_ERR_SELF_CHECK: return "zkattest: proof failed its self-check";
    default: return "zkattest: internal status";
  }
}

struct Params : public Napi::ObjectWrap<Params> {
  zka_params* h = nullptr;
  static Napi::FunctionReference ctor;
  static Napi::Function Init(Napi::Env env) {
    Napi::Function f = DefineClass(env, "Params", {});
    ctor = Napi::Persistent(f);
    ctor.SuppressDestruct();
    return f;
  }
  explicit Params(const Napi::CallbackInfo& info) : Napi::ObjectWrap<Params>(info) {}
  ~Params() { release(); }
  void release() {
    if (!h) return;
    std::lock_guard<std::mutex> lk(g_mu);
    zka_params_destroy(h);
    h = nullptr;
  }
};
Napi::FunctionReference Params::ctor;

template <class T>
std::vector<T> to_vec(const Napi::Value& v) {
  auto a = v.As<Napi::TypedArrayOf<T>>();
  return std::vector<T>(a.Data(), a.Data() + a.ElementLength());
}

class ProveWorker : public Napi::AsyncWorker {
 public:
  ProveWorker(Napi::Env env, zka_params* p, std::vector<uint8_t> msg, std::vector<uint8_t> sig, std::vector<uint8_t> pk,
              std::vector<uint32_t> which, std::vector<uint8_t> ring, std::vector<uint8_t> tape, uint32_t sec)
      : Napi::AsyncWorker(env), deferred(Napi::Promise::Deferred::New(env)), p_(p), msg_(std::move(msg)), sig_(std::move(sig)),
        pk_(std::move(pk)), which_(std::move(which)), ring_(std::move(ring)), tape_(std::move(tape)), sec_(sec) {}
  void Execute() override {
    const uint32_t B = (uint32_t)which_.size(), N = (uint32_t)(ring_.size() / 32);
    if (B == 0) return;
    if (!p_ || msg_.size() != (size_t)B * 32 || sig_.size() != (size_t)B * 64 || pk_.size() != (size_t)B * 65 || tape_.size() % B) {
      SetError("zkattest: proveBatch argument sizes");
      return;
    }
    stride_ = zka_proof_max_len(N, sec_);
    proofs_.resize((size_t)B * stride_);
    lens_.resize(B);
    status_.resize(B);
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = zka_prove_batch(g_ctx, p_, B, msg_.data(), sig_.data(), pk_.data(), which_.data(), ring_.data(), N, tape_.data(),
                             tape_.size() / B, proofs_.data(), stride_, lens_.data(), status_.data());
    if (rc != 0) SetError(zka_last_error(g_ctx));
  }
  void OnOK() override {
    Napi::Env env = Env();
    for (size_t i = 0; i < status_.size(); i++)
      if (status_[i] != 0) { deferred.Reject(Napi::Error::New(env, status_message(status_[i])).Value()); return; }
    Napi::Object o = Napi::Object::New(env);
    o.Set("proofs", Napi::Buffer<uint8_t>::Copy(env, proofs_.data(), proofs_.size()));
    o.Set("stride", Napi::Number::New(env, (double)stride_));
    o.Set("lens", Napi::Buffer<uint32_t>::Copy(env, lens_.data(), lens_.size()));
    deferred.Resolve(o);
  }
  void OnError(const Napi::Error& e) override { deferred.Reject(e.Value()); }
  Napi::Promise::Deferred deferred;

 private:
  zka_params* p_;
  std::vector<uint8_t> msg_, sig_, pk_;
  std::vector<uint32_t> which_;
  std::vector<uint8_t> ring_, tape_, proofs_;
  std::vector<uint32_t> lens_;
  std::vector<int32_t> status_;
  uint32_t sec_;
  size_t stride_ = 0;
};

class VerifyWorker : public Napi::AsyncWorker {
 public:
  VerifyWorker(Napi::Env env, zka_params* p, std::vector<uint8_t> msg, std::vector<uint8_t> ring, std::vector<uint8_t> proofs,
               std::vector<uint32_t> lens, size_t stride, std::vector<uint8_t> tape, uint32_t sec)
      : Napi::AsyncWorker(env), deferred(Napi::Promise::Deferred::New(env)), p_(p), msg_(std::move(msg)), ring_(std::move(ring)),
        proofs_(std::move(proofs)), lens_(std::move(lens)), tape_(std::move(tape)), stride_(stride), sec_(sec) {}
  void Execute() override {
    const uint32_t B = (uint32_t)lens_.size(), N = (uint32_t)(ring_.size() / 32);
    if (B == 0) return;
    if (!p_ || msg_.size() != (size_t)B * 32 || proofs_.size() < (size_t)B * stride_ || tape_.size() % B) {
      SetError("zkattest: verifyBatch argument sizes");
      return;
    }
    ok_.resize(B);
    status_.resize(B);
    std::lock_guard<std::mutex> lk(g_mu);
    int rc = zka_verify_batch(g_ctx, p_, B, msg_.data(), ring_.data(), N, proofs_.data(), stride_, lens_.data(), tape_.data(),
                              tape_.size() / B, ok_.data(), status_.data());
    if (rc != 0) SetError(zka_last_error(g_ctx));   // e.g. 'security level not achieved' (exp.ts:244)
  }
  void OnOK() override {
    Napi::Env env = Env();
    for (size_t i = 0; i < status_.size(); i++)
      if (status_[i] != 0) { deferred.Reject(Napi::Error::New(env, status_message(status_[i])).Value()); return; }
    Napi::Object o = Napi::Object::New(env);
    o.Set("ok", Napi::Buffer<uint8_t>::Copy(env, ok_.data(), ok_.size()));
    deferred.Resolve(o);
  }
  void OnError(const Napi::Error& e) override { deferred.Reject(e.Value()); }
  Napi::Promise::Deferred deferred;

 private:
  zka_params* p_;
  std::vector<uint8_t> msg_, ring_, proofs_;
  std::vector<uint32_t> lens_;
  std::vector<uint8_t> tape_, ok_;
  std::vector<int32_t> status_;
  size_t stride_;
  uint32_t sec_;
};

class KeyToIntWorker : public Napi::AsyncWorker {
 public:
  KeyToIntWorker(Napi::Env env, std::vector<uint8_t> pk)
      : Napi::AsyncWorker(env), deferred(Napi::Promise::Deferred::New(env)), pk_(std::move(pk)) {}
  void Execute() override {
    const uint32_t count = (uint32_t)(pk_.size() / 65);
    if (count == 0 || pk_.size() % 65) { SetError("invalid public key"); return; }
    x_.resize((size_t)count * 32);
    status_.resize(count);
    std::lock_guard<std::mutex> lk(g_mu);
    if (zka_key_to_int(g_ctx, count, pk_.data(), x_.data(), status_.data()) != 0) SetError(zka_last_error(g_ctx));
  }
  void OnOK() override {
    Napi::Env env = Env();
    for (int32_t s : status_)
      if (s != 0) { deferred.Reject(Napi::Error::New(env, status_message(s)).Value()); return; }
    deferred.Resolve(Napi::Buffer<uint8_t>::Copy(env, x_.data(), x_.size()));
  }
  void OnError(const Napi::Error& e) override { deferred.Reject(e.Value()); }
  Napi::Promise::Deferred deferred;

 private:
  std::vector<uint8_t> pk_, x_;
  std::vector<int32_t> status_;
};

zka_params* unwrap_params(const Napi::Value& v) {
  Params* P = Napi::ObjectWrap<Params>::Unwrap(v.As<Napi::Object>());
  return P ? P->h : nullptr;
}

Napi::Value ProveBatch(const Napi::CallbackInfo& info) {
  auto* w = new ProveWorker(info.Env(), unwrap_params(info[0]), to_vec<uint8_t>(info[1]), to_vec<uint8_t>(info[2]),
                            to_vec<uint8_t>(info[3]), to_vec<uint32_t>(info[4]), to_vec<uint8_t>(info[5]), to_vec<uint8_t>(info[6]),
                            info[7].As<Napi::Number>().Uint32Value());
  w->Queue();
  return w->deferred.Promise();
}
Napi::Value VerifyBatch(const Napi::CallbackInfo& info) {
  auto* w = new VerifyWorker(info.Env(), unwrap_params(info[0]), to_vec<uint8_t>(info[1]), to_vec<uint8_t>(info[2]),
                             to_vec<uint8_t>(info[3]), to_vec<uint32_t>(info[4]), (size_t)info[5].As<Napi::Number>().Int64Value(),
                             to_vec<uint8_t>(info[6]), info[7].As<Napi::Number>().Uint32Value());
  w->Queue();
  return w->deferred.Promise();
}
Napi::Value KeyToInt(const Napi::CallbackInfo& info) {
  auto* w = new KeyToIntWorker(info.Env(), to_vec<uint8_t>(info[0]));
  w->Queue();
  return w->deferred.Promise();
}

Napi::Value ParamsGenerate(const Napi::CallbackInfo& info) {
  auto rnd = info[0].As<Napi::Uint8Array>();
  uint8_t hn[65], hp[67];
  int wp = 67;   // ProofGroup point bytes of the linked library: 67 (libzkattest.so) or 65 (libzkattest_war256.so)
  zka_proof_group(nullptr, 0, &wp, nullptr);
  int rc;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    rc = rnd.ElementLength() == 64 ? zka_params_generate(g_ctx, rnd.Data(), hn, hp) : ZKA_E_ARG;
  }
  if (rc != 0) {
    Napi::Error::New(info.Env(), rc == ZKA_E_ARG ? "zkattest: paramsGenerate needs 64 bytes of randomness" : zka_last_error(g_ctx))
        .ThrowAsJavaScriptException();
    return info.Env().Undefined();
  }
  Napi::Object o = Napi::Object::New(info.Env());
  o.Set("hNist", Napi::Buffer<uint8_t>::Copy(info.Env(), hn, 65));
  o.Set("hProof", Napi::Buffer<uint8_t>::Copy(info.Env(), hp, (size_t)wp));
  return o;
}
// SystemParametersList -> device tables (zka_params_create): synchronous, ~0.2 s, once per parameter set
Napi::Value ParamsCreate(const Napi::CallbackInfo& info) {
  auto hn = info[0].As<Napi::Uint8Array>();
  auto hp = info[1].As<Napi::Uint8Array>();
  const uint32_t sec = info[2].As<Napi::Number>().Uint32Value();
  int wp = 67;
  zka_proof_group(nullptr, 0, &wp, nullptr);
  if (hn.ElementLength() != 65 || hp.ElementLength() != (size_t)wp) {
    Napi::Error::New(info.Env(), "error deserializing Point").ThrowAsJavaScriptException();
    return info.Env().Undefined();
  }
  zka_params* h = nullptr;
  int rc;
  {
    std::lock_guard<std::mutex> lk(g_mu);
    rc = zka_params_create(g_ctx, hn.Data(), hp.Data(), sec, &h);
  }
  if (rc != 0) {
    Napi::Error::New(info.Env(), zka_last_error(g_ctx)).ThrowAsJavaScriptException();
    return info.Env().Undefined();
  }
  Napi::Object o = Params::ctor.New({});
  Napi::ObjectWrap<Params>::Unwrap(o)->h = h;
  return o;
}
Napi::Value ParamsDestroy(const Napi::CallbackInfo& info) {
  Params* P = Napi::ObjectWrap<Params>::Unwrap(info[0].As<Napi::Object>());
  if (P) P->release();
  return info.Env().Undefined();
}

Napi::Object InitAll(Napi::Env env, Napi::Object exports) {
  if (zka_init(0, &g_ctx) != 0) {
    Napi::Error::New(env, "zkattest: no CUDA device (no CPU fallback)").ThrowAsJavaScriptException();
    return exports;
  }
  exports.Set("Params", Params::Init(env));
  exports.Set("paramsGenerate", Napi::Function::New(env, ParamsGenerate));
  exports.Set("paramsCreate", Napi::Function::New(env, ParamsCreate));
  exports.Set("paramsDestroy", Napi::Function::New(env, ParamsDestroy));
  exports.Set("keyToInt", Napi::Function::New(env, KeyToInt));
  exports.Set("proveBatch", Napi::Function::New(env, ProveBatch));
  exports.Set("verifyBatch", Napi::Function::New(env, VerifyBatch));
  return exports;
}

}  // namespace

#ifndef ZKA_NAPI_MODULE
#define ZKA_NAPI_MODULE zkattest   // binding.gyp builds the same source a second time as zkattest_war256
#endif
NODE_API_MODULE(ZKA_NAPI_MODULE, InitAll)
