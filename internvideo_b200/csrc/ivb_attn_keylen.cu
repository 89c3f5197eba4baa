// ivb_attn_keylen.cu — the attention forward with per-clip key lengths (ivb_attn_fwd_keylen): the key-padding mask of
// right-padded text, the reference's additive -10000 on the padded keys of BERT captions
// (InternVideo2/multi_modality/models/backbones/bert/xbert.py:1099-1119).  The kernel is ivb_attn_fwd.cuh's attn_fwd
// with its KEYLEN switch; it has its own translation unit so that the objects of the other attention kernels keep
// their instantiations.
#include "ivb_attn_fwd.cuh"

namespace ivb {

// kv_len: int32 [B], the keys each clip keeps
template <int KA, int NO, int KS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
attn_fwd_keylen_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p, const int* kv_len) {
  attn_fwd<AttnElt::BF16, KA, NO, KS, false, false, true>(tmQ, tmK, tmV, p, nullptr, kv_len);
}

}  // namespace ivb

using namespace ivb;

extern "C" int ivb_attn_fwd_keylen(const void* q, long ldq, const void* k, long ldk, const void* v, long ldv, void* out,
                                   long ldo, float* lse2, int B, int n, int H, int d, float softmax_scale,
                                   const int* kv_len, void* stream) {
  if (kv_len == nullptr) return set_error("ivb_attn_fwd_keylen: kv_len is null");
  return attn_fwd_setup("ivb_attn_fwd_keylen", q, ldq, k, ldk, v, ldv, out, ldo, lse2, B, n, H, d, softmax_scale,
                        [&](auto hd, const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv,
                            const AttnFwdParams& p) {
    return launch_attn<attn_fwd_keylen_kernel<hd.KA, hd.NO, hd.KS>, NO_PDL>(
        "cudaFuncSetAttribute(attn_fwd_keylen)", "attn_fwd_keylen_kernel", FwdSmem<hd.KA>::BYTES, B, n, H,
        reinterpret_cast<cudaStream_t>(stream), tq, tk, tv, p, kv_len);
  });
}
