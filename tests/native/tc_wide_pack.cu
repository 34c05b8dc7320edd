// tcw_plan_decoder on the host, without a device: a plain decoder with a 512-wide layer, a 256-wide one and a latent_in
// concat (layer widths 67 -> 320 -> 253 (+67) -> 512 -> 200 -> 1).  Reads the layers' weights (row-major [out][in],
// float32, layer after layer) from argv[1] and writes to argv[2]:  int32 n_steps, n_fwd, then per step kind, n_mma,
// k_steps, w_off, layer, n_real, cat_off, mask_layer;  int64 blob bytes; the blob.  Also checks that tc_pack_decoder
// declines the decoder.  Prints "packed" and exits 0 on success.
#include <cstdio>
#include <string>
#include <vector>

#include "dspgn_common.cuh"
#include "dspgn_simt.cuh"
#include "dspgn_solve.cuh"
#include "dspgn_tc.cuh"
#include "dspgn_tc_wide.cuh"

using namespace dspgn;

int main(int argc, char** argv) {
  if (argc != 3) return 2;
  const int nl = 5, in_dim[nl] = {67, 320, 320, 512, 200}, out_dim[nl] = {320, 253, 512, 200, 1};
  DspgnDecoderSpec spec{};
  spec.num_linear = nl; spec.latent_size = 64; spec.latent_in_layer = 2;
  DecoderDev dv{};
  dv.L = 64; dv.n_lin = nl; dv.in0 = 67; dv.latent_in = 2; dv.generic = 0;
  std::vector<std::vector<float>> w(nl), b(nl);
  std::vector<const float*> W(nl), B(nl);
  FILE* f = std::fopen(argv[1], "rb");
  if (!f) return 3;
  for (int k = 0; k < nl; ++k) {
    spec.in_dim[k] = dv.in_dim[k] = in_dim[k]; spec.out_dim[k] = dv.out_dim[k] = out_dim[k];
    w[k].resize((size_t)in_dim[k] * out_dim[k]); b[k].assign(out_dim[k], 0.f);
    if (std::fread(w[k].data(), sizeof(float), w[k].size(), f) != w[k].size()) return 4;
    W[k] = w[k].data(); B[k] = b[k].data();
  }
  std::fclose(f);
  TcDecoderHost h;
  DecoderDev dt = dv;
  std::string err;
  if (tc_pack_decoder(spec, W.data(), B.data(), h, &dt, err) != 0 || h.ok) { std::printf("tc_pack_decoder packed it\n"); return 5; }
  TcPlan P;
  std::vector<unsigned char> blob;
  if (!tcw_plan_decoder(dv, W.data(), P, blob)) { std::printf("declined\n"); return 6; }
  FILE* o = std::fopen(argv[2], "wb");
  if (!o) return 7;
  std::vector<int> hdr = {P.n_steps, P.n_fwd};
  for (int s = 0; s < P.n_steps; ++s) {
    const TcStep& t = P.step[s];
    for (int v : {t.kind, t.n_mma, t.k_steps, (int)t.w_off, t.layer, t.n_real, t.cat_off, t.mask_layer}) hdr.push_back(v);
  }
  const long long n = (long long)blob.size();
  std::fwrite(hdr.data(), sizeof(int), hdr.size(), o);
  std::fwrite(&n, sizeof(n), 1, o);
  std::fwrite(blob.data(), 1, blob.size(), o);
  std::fclose(o);
  std::printf("packed\n");
  return 0;
}
