// Microbenchmark: what do the pieces of the solver's iteration graph cost on this GPU?
//   chain of dependent small kernels, IF node (not taken), WHILE node with one trip, a WHILE node that loops
//   on the device, and back-to-back launches of a one-kernel graph.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o graph_overheads graph_overheads.cu
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

__global__ void small_kernel(float* p, int n) {   // the shape of the solver's vector passes: 137 x 256, 1 float4 per thread
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { float4 v = reinterpret_cast<float4*>(p)[i]; v.x += 1.0f; reinterpret_cast<float4*>(p)[i] = v; }
}
__global__ void set_cond(cudaGraphConditionalHandle h, unsigned v) { if (threadIdx.x == 0) cudaGraphSetConditional(h, v); }
__global__ void small_kernel_setting(float* p, int n, cudaGraphConditionalHandle h, unsigned v) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { float4 t = reinterpret_cast<float4*>(p)[i]; t.x += 1.0f; reinterpret_cast<float4*>(p)[i] = t; }
  if (i == 0) cudaGraphSetConditional(h, v);
}
__global__ void loop_counter(int* c, int limit, cudaGraphConditionalHandle h) {
  if (threadIdx.x == 0) { int v = *c + 1; *c = v; cudaGraphSetConditional(h, v < limit ? 1u : 0u); }
}
__global__ void reset_counter(int* c, cudaGraphConditionalHandle h) { if (threadIdx.x == 0) { *c = 0; cudaGraphSetConditional(h, 1u); } }

static const int NB = 137, NT = 256, N4 = 137 * 256;
static float* buf;
static int* counter;
static cudaStream_t cap, cap2;

static void k(cudaStream_t st) { small_kernel<<<NB, NT, 0, st>>>(buf, N4); }

static cudaGraphNode_t add_cond(cudaStream_t st, cudaGraphConditionalHandle h, cudaGraphConditionalNodeType type, cudaGraph_t* body) {
  cudaStreamCaptureStatus cs; cudaGraph_t cg; const cudaGraphNode_t* deps; size_t nd;
  CK(cudaStreamGetCaptureInfo_v2(st, &cs, nullptr, &cg, &deps, &nd));
  cudaGraphNodeParams np = {};
  np.type = cudaGraphNodeTypeConditional;
  np.conditional.handle = h; np.conditional.type = type; np.conditional.size = 1;
  cudaGraphNode_t node;
  CK(cudaGraphAddNode(&node, cg, deps, nd, &np));
  *body = np.conditional.phGraph_out[0];
  CK(cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));
  return node;
}
static cudaGraphConditionalHandle new_handle(cudaStream_t st) {
  cudaStreamCaptureStatus cs; cudaGraph_t cg; const cudaGraphNode_t* deps; size_t nd;
  CK(cudaStreamGetCaptureInfo_v2(st, &cs, nullptr, &cg, &deps, &nd));
  cudaGraphConditionalHandle h;
  CK(cudaGraphConditionalHandleCreate(&h, cg, 0, cudaGraphCondAssignDefault));
  return h;
}

static double time_graph(cudaGraphExec_t ex, int launches) {
  cudaStream_t st; CK(cudaStreamCreate(&st));
  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int i = 0; i < 20; ++i) CK(cudaGraphLaunch(ex, st));
  CK(cudaStreamSynchronize(st));
  double best = 1e30;
  for (int rep = 0; rep < 5; ++rep) {
    CK(cudaEventRecord(a, st));
    for (int i = 0; i < launches; ++i) CK(cudaGraphLaunch(ex, st));
    CK(cudaEventRecord(b, st));
    CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    double us = 1e3 * ms / launches;
    if (us < best) best = us;
  }
  CK(cudaStreamDestroy(st));
  return best;
}

template <class F> static cudaGraphExec_t build(F f) {
  cudaGraph_t g; cudaGraphExec_t ex;
  CK(cudaStreamBeginCapture(cap, cudaStreamCaptureModeRelaxed));
  f();
  CK(cudaStreamEndCapture(cap, &g));
  CK(cudaGraphInstantiate(&ex, g, 0));
  return ex;
}

int main() {
  CK(cudaMalloc(&buf, sizeof(float4) * N4)); CK(cudaMemset(buf, 0, sizeof(float4) * N4));
  CK(cudaMalloc(&counter, sizeof(int)));
  CK(cudaStreamCreateWithFlags(&cap, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&cap2, cudaStreamNonBlocking));
  const int L = 300;

  auto g1 = build([&] { k(cap); });
  auto g8 = build([&] { for (int i = 0; i < 8; ++i) k(cap); });
  auto g32 = build([&] { for (int i = 0; i < 32; ++i) k(cap); });
  double t1 = time_graph(g1, L), t8 = time_graph(g8, L), t32 = time_graph(g32, L);
  printf("graph of 1 kernel              %7.2f us per launch\n", t1);
  printf("graph of 8 dependent kernels   %7.2f us per launch  => %.2f us per extra kernel node\n", t8, (t8 - t1) / 7);
  printf("graph of 32 dependent kernels  %7.2f us per launch  => %.2f us per extra kernel node\n", t32, (t32 - t8) / 24);

  // 8 kernels + gate kernel + IF node (never taken) in the middle
  auto gif = build([&] {
    cudaGraphConditionalHandle h = new_handle(cap);
    for (int i = 0; i < 4; ++i) k(cap);
    set_cond<<<1, 32, 0, cap>>>(h, 0u);
    cudaGraph_t body; add_cond(cap, h, cudaGraphCondTypeIf, &body);
    CK(cudaStreamBeginCaptureToGraph(cap2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    k(cap2); CK(cudaStreamEndCapture(cap2, nullptr));
    for (int i = 0; i < 4; ++i) k(cap);
  });
  double tif = time_graph(gif, L);
  printf("8 kernels + gate kernel + IF(not taken)   %7.2f us  => gate + IF = %.2f us\n", tif, tif - t8);
  // same, the IF handle set by the preceding vector kernel (no separate gate)
  auto gif2 = build([&] {
    cudaGraphConditionalHandle h = new_handle(cap);
    for (int i = 0; i < 3; ++i) k(cap);
    small_kernel_setting<<<NB, NT, 0, cap>>>(buf, N4, h, 0u);
    cudaGraph_t body; add_cond(cap, h, cudaGraphCondTypeIf, &body);
    CK(cudaStreamBeginCaptureToGraph(cap2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    k(cap2); CK(cudaStreamEndCapture(cap2, nullptr));
    for (int i = 0; i < 4; ++i) k(cap);
  });
  double tif2 = time_graph(gif2, L);
  printf("8 kernels + IF(not taken), no gate        %7.2f us  => IF alone = %.2f us\n", tif2, tif2 - t8);
  // IF taken, body of 1 kernel
  auto gif3 = build([&] {
    cudaGraphConditionalHandle h = new_handle(cap);
    for (int i = 0; i < 3; ++i) k(cap);
    small_kernel_setting<<<NB, NT, 0, cap>>>(buf, N4, h, 1u);
    cudaGraph_t body; add_cond(cap, h, cudaGraphCondTypeIf, &body);
    CK(cudaStreamBeginCaptureToGraph(cap2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    k(cap2); CK(cudaStreamEndCapture(cap2, nullptr));
    for (int i = 0; i < 4; ++i) k(cap);
  });
  double tif3 = time_graph(gif3, L);
  printf("8 kernels + IF(taken, 1 kernel body)      %7.2f us  => IF taken overhead = %.2f us over 9 chained kernels\n", tif3, tif3 - t8 - (t8 - t1) / 7);

  // 5 kernels, WHILE node whose 3-kernel body runs exactly once, 1 kernel  (the solver's shape)
  auto gwh = build([&] {
    cudaGraphConditionalHandle h = new_handle(cap);
    for (int i = 0; i < 3; ++i) k(cap);
    small_kernel_setting<<<NB, NT, 0, cap>>>(buf, N4, h, 1u);
    cudaGraph_t body; add_cond(cap, h, cudaGraphCondTypeWhile, &body);
    CK(cudaStreamBeginCaptureToGraph(cap2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    k(cap2); k(cap2); small_kernel_setting<<<NB, NT, 0, cap2>>>(buf, N4, h, 0u);
    CK(cudaStreamEndCapture(cap2, nullptr));
    k(cap);
  });
  double twh = time_graph(gwh, L);
  printf("4 kernels + WHILE(3-kernel body, 1 trip) + 1 kernel  %7.2f us  => WHILE node overhead = %.2f us over 8 chained kernels\n", twh, twh - t8);

  // a WHILE node looping 64 times over a 5-kernel body: per-trip cost
  for (int body_k : {3, 5}) {
    auto gl = build([&] {
      cudaGraphConditionalHandle h = new_handle(cap);
      reset_counter<<<1, 32, 0, cap>>>(counter, h);
      cudaGraph_t body; add_cond(cap, h, cudaGraphCondTypeWhile, &body);
      CK(cudaStreamBeginCaptureToGraph(cap2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
      for (int i = 0; i < body_k - 1; ++i) k(cap2);
      loop_counter<<<1, 32, 0, cap2>>>(counter, 64, h);
      CK(cudaStreamEndCapture(cap2, nullptr));
    });
    double tl = time_graph(gl, 20);
    printf("WHILE looping 64 x (%d kernels, last one 1 thread)   %7.2f us per trip  (chain of %d kernels = %.2f us)\n",
           body_k, tl / 64, body_k, body_k * (t8 - t1) / 7);
  }
  return 0;
}
