// libb200tts.so -- the kernels of the Tacotron decoder sessions (b200tts_taco_session_*, whose host side is in tacotron.cu).
//
// Their own translation unit, like every model stage's (build.py): the session instantiation of taco_decoder_run cannot change
// the code ptxas gives the batch decoders in tacotron.cu.  Like tacotron.cu's, the `sm` array asks for a 1024-byte base.
#include <algorithm>

#include "api.h"
#include "taco_decoder_body.cuh"

namespace b200tts {

// a slice of decoder sessions: CTA u resumes S.row[u] (see TacoSessRow), always on the biased body (a bias of 0 is the unbiased
// decoder bit for bit), with the row's own window flag and Philox key
__global__ void __launch_bounds__(kTacoThreads, 1) taco_decoder_session_kernel(TacoWeights W, const __grid_constant__ TacoSessIO S) {
  const TacoSessRow& r = S.row[blockIdx.x];
  TacoArgs a{};
  a.memory = r.memory; a.keys = r.keys; a.lengths = &r.Tx;
  a.B = 1; a.Tx_max = r.Tx; a.max_steps = r.pos + r.n; a.window = r.window;
  a.rng_mode = 0; a.seed = r.seed; a.utt_offset = r.id;
  a.frames = r.frames; a.stop = r.stop; a.nsteps = r.status;
  taco_decoder_run<false, true, true>(W, a, TacoGtaArgs{}, &r.mu_bias, &r);
}

void launch_taco_sessions(const TacoWeights& W, const TacoSessIO& io, int rows, size_t smem, cudaStream_t st) {
  B200_CUDA(cudaFuncSetAttribute(taco_decoder_session_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  taco_decoder_session_kernel<<<rows, kTacoThreads, smem, st>>>(W, io);
  B200_CUDA(cudaGetLastError());
}

// Row i: the first pos[i] frames / stop values of session i, then zeros up to T_max.
__global__ void taco_session_outputs_kernel(const __grid_constant__ TacoSessOut g, int T_max, int M, float* __restrict__ frames,
                                            float* __restrict__ stop, int32_t* __restrict__ nsteps) {
  const int i = blockIdx.y, pos = g.pos[i];
  const size_t nf = (size_t)T_max * M;
  for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < nf; e += (size_t)gridDim.x * blockDim.x)
    frames[(size_t)i * nf + e] = e < (size_t)pos * M ? g.frames[i][e] : 0.f;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < T_max; t += gridDim.x * blockDim.x)
    stop[(size_t)i * T_max + t] = t < pos ? g.stop[i][t] : 0.f;
  if (blockIdx.x == 0 && threadIdx.x == 0) nsteps[i] = pos;
}

void launch_taco_session_outputs(const TacoSessOut& g, int n, int T_max, int M, float* frames, float* stop, int32_t* nsteps,
                                 cudaStream_t st) {
  const unsigned gx = (unsigned)std::min<size_t>(((size_t)T_max * M + 255) / 256, 64);
  taco_session_outputs_kernel<<<dim3(gx, n), 256, 0, st>>>(g, T_max, M, frames, stop, nsteps);
  B200_CUDA(cudaGetLastError());
}

}  // namespace b200tts
