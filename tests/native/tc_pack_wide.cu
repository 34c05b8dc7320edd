// tc_pack_decoder on decoder shapes without a device: a plain decoder with 512-wide layers (DeepSDF's 8 x 512 network)
// is declined (TcDecoderHost.ok stays false, no weight image is packed) before any CUDA call, so the solver falls back
// to the SIMT engine instead of packing wgmma images truncated to N = 256.  Prints "declined" and exits 0 on success.
#include <cstdio>
#include <string>
#include <vector>

#include "dspgn_common.cuh"
#include "dspgn_simt.cuh"
#include "dspgn_solve.cuh"
#include "dspgn_tc.cuh"

using namespace dspgn;

int main() {
  for (int width : {512, 257}) {
    DspgnDecoderSpec spec{};
    spec.num_linear = 9; spec.latent_size = 64; spec.latent_in_layer = 4;
    for (int k = 0; k < 9; ++k) {
      spec.in_dim[k] = (k == 0) ? 67 : width;             // layer 4: (width - 67) + the 67 inputs
      spec.out_dim[k] = (k == 8) ? 1 : (k == 3 ? width - 67 : width);
    }
    std::vector<std::vector<float>> w(9), b(9);
    std::vector<const float*> W(9), B(9);
    for (int k = 0; k < 9; ++k) {
      w[k].assign((size_t)spec.in_dim[k] * spec.out_dim[k], 0.01f); b[k].assign(spec.out_dim[k], 0.f);
      W[k] = w[k].data(); B[k] = b[k].data();
    }
    DecoderDev dv{};
    dv.latent_in = 4;
    TcDecoderHost h;
    std::string err;
    const int rc = tc_pack_decoder(spec, W.data(), B.data(), h, &dv, err);
    if (rc != 0 || h.ok || h.blob != nullptr || dv.tc_blob != nullptr) {
      std::printf("width %d: rc %d ok %d blob %p (%s)\n", width, rc, (int)h.ok, h.blob, err.c_str());
      return 1;
    }
  }
  std::printf("declined\n");
  return 0;
}
