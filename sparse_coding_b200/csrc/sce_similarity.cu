// sce_similarity.cu — dictionary similarity (sce_similarity): cosine maxima and capacity over a list of dictionary
// pairs, on the split-operand GEMM.
#include <vector>

#include "sce_engine.cuh"

// maxima keys (EpiSimilarity) -> floats, in place; key 0 (no valid entry: an atom beyond rows[m]) becomes NaN
__global__ void key_to_float_kernel(uint32_t* __restrict__ v, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t k = v[i];
    v[i] = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
  }
}

// capacity_per_feature (standard_metrics.py:356-362) of every self-pair (m, m): diag(S^2) / rowsum(S^2), the row sum
// taken over the partials of EpiSimilarity in a fixed order. Atoms beyond rows[m] get NaN. A zero row gives 0 / 0 = NaN,
// as in the reference.
__global__ void capacity_kernel(const int* __restrict__ pairs, const int* __restrict__ rows, const float* __restrict__ sq_part,
                                const float* __restrict__ diag, int na, int parts, float* __restrict__ out) {
  const int q = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = pairs[2 * q];
  if (i >= na || m != pairs[2 * q + 1]) return;
  float* o = out + (long long)m * na + i;
  if (i >= rows[m]) {
    *o = __int_as_float(0x7FFFFFFF);
    return;
  }
  const float* s = sq_part + ((long long)q * na + i) * parts;
  float sum = 0.f;
  for (int t = 0; t < parts; ++t) sum += s[t];
  const float dg = diag[(long long)q * na + i];
  *o = dg * dg / sum;
}

struct SimOperand {   // one side of sce_similarity
  const float* w;
  int models, rows;
  int normalize;
  float floor;
};

// Workspace of one call: operand planes (4 B per element), the pair list and valid-row counts, the range flags of the
// f16f8 split, and (capacity) the sum-of-squares partials [P][na][2 tiles_n] and diagonal [P][na]. With base == nullptr
// only measures; `f8` only changes the order of the planes, not the bytes.
struct SimCarve {
  Planes a, b;
  int *pairs, *a_rows, *b_rows;
  uint32_t* flags;
  float *sq_part, *diag;
};
static size_t sim_carve(uint8_t* base, bool f8, long long ma, long long na, long long mb, long long nb, long long d,
                        long long n_pairs, bool capacity, SimCarve* out) {
  Carve c{base, 0};
  SimCarve s{};
  s.a = c.planes((size_t)(ma * na * d), f8);
  if (mb > 0) s.b = c.planes((size_t)(mb * nb * d), f8);
  s.pairs = c.take<int>((size_t)(2 * n_pairs));
  s.a_rows = c.take<int>((size_t)ma);
  s.b_rows = mb > 0 ? c.take<int>((size_t)mb) : s.a_rows;
  s.flags = c.take<uint32_t>(kFlagWords);
  if (capacity) {
    const long long tiles_n = (na + kBN - 1) / kBN;
    s.sq_part = c.take<float>((size_t)(n_pairs * na * 2 * tiles_n));
    s.diag = c.take<float>((size_t)(n_pairs * na));
  }
  if (out) *out = s;
  return align_up(c.off, 1024);
}
static size_t sim_workspace(long long ma, long long na, long long mb, long long nb, long long d, long long n_pairs, bool capacity) {
  const size_t a = sim_carve(nullptr, false, ma, na, mb, nb, d, n_pairs, capacity, nullptr);
  const size_t b = sim_carve(nullptr, true, ma, na, mb, nb, d, n_pairs, capacity, nullptr);
  return a > b ? a : b;
}

// fp32 operand -> planes: normalised rows (dict_rows_kernel<MODE_PREPARE>, LearnedDict.get_learned_dict) or the matrix
// as given (split_rows_kernel; f16f8: sets the range flags when a value does not fit fp16)
template <int AR>
static int sim_planes(Launcher& L, const SimOperand& o, int d, const Planes& w, uint32_t* flags) {
  const long long rows = (long long)o.models * o.rows;
  if (o.normalize)
    return launch_dict_rows_t<MODE_PREPARE, AR>(L, const_cast<float*>(o.w), nullptr, nullptr, nullptr, w, nullptr, rows, d,
                                                 1, o.floor, AdamHyper{}, nullptr, nullptr);
  return launch_split_rows<AR>(L, o.w, w, rows * d / 4, AR == kArithF16F8 ? flags : nullptr);
}

template <int AR>
static int run_similarity_t(Launcher& L, const SimOperand& A, const SimOperand& B, bool b_is_a, int d, int n_pairs,
                            const SimCarve& w, float* row_max, float* col_max, float* capacity, int device, int sms) {
  TRY(sim_planes<AR>(L, A, d, w.a, w.flags));
  if (!b_is_a) TRY(sim_planes<AR>(L, B, d, w.b, w.flags));
  // both operands are dictionary rows, K-major over d: the encode GEMM's B-operand geometry on both sides
  GemmMaps maps{};
  bool ok = operand_maps(maps.a[0], w.a, A.models, A.rows, d, (uint64_t)A.rows * d, kBM, gemm_bk(AR));
  ok = ok && operand_maps(maps.b[0], b_is_a ? w.a : w.b, B.models, B.rows, d, (uint64_t)B.rows * d, kBN, gemm_bk(AR));
  if (!ok) return fail(SCE_ERR_CUDA, "cuTensorMapEncodeTiled failed (similarity: na=%d, nb=%d, d=%d)", A.rows, B.rows, d);
  const int tiles_n = (B.rows + kBN - 1) / kBN;
  const EpiSimilarity::Params ep{w.pairs, w.a_rows, w.b_rows, reinterpret_cast<uint32_t*>(row_max),
                                 reinterpret_cast<uint32_t*>(col_max), capacity ? w.sq_part : nullptr, w.diag, tiles_n};
  if (row_max) CUDA_TRY(cudaMemsetAsync(row_max, 0, (size_t)n_pairs * A.rows * sizeof(float), L.st));
  if (col_max) CUDA_TRY(cudaMemsetAsync(col_max, 0, (size_t)n_pairs * B.rows * sizeof(float), L.st));
  TRY((launch_gemm_t<EpiSimilarity, false, false, false, AR, AR == kArithF16F8>(L, n_pairs, device, sms, maps, 1, kOnes,
                                                                                  kOnes, d, 3, A.rows, B.rows, ep)));
  auto to_float = [&](float* v, long long n) {
    const int blocks = (int)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024);
    return L.launch(key_to_float_kernel, blocks, 256, 0, reinterpret_cast<uint32_t*>(v), n);
  };
  if (row_max) TRY(to_float(row_max, (long long)n_pairs * A.rows));
  if (col_max) TRY(to_float(col_max, (long long)n_pairs * B.rows));
  if (!capacity) return SCE_OK;
  return L.launch(capacity_kernel, dim3((A.rows + 255) / 256, n_pairs), 256, 0, w.pairs, w.a_rows, w.sq_part, w.diag,
                  A.rows, 2 * tiles_n, capacity);
}

extern "C" {

size_t sce_similarity_workspace_bytes(int ma, int na, int mb, int nb, int d, int n_pairs, int want_capacity) {
  if (ma < 1 || na < 1 || mb < 0 || (mb > 0 && nb < 1) || d < 8 || n_pairs < 1) return 0;
  return sim_workspace(ma, na, mb, mb > 0 ? nb : 0, d, n_pairs, want_capacity != 0);
}

int sce_similarity(const float* a, int ma, int na, const int* a_rows, float a_norm_floor, int a_normalize,
                   const float* b, int mb, int nb, const int* b_rows, float b_norm_floor, int b_normalize,
                   int d, const int* pairs, int n_pairs, int arith, float* row_max, float* col_max, float* capacity,
                   void* workspace, size_t workspace_bytes, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!a) return fail(SCE_ERR_INVALID, "similarity: a is NULL");
  if (ma < 1 || na < 1) return fail(SCE_ERR_INVALID, "similarity: ma (%d) and na (%d) must be >= 1", ma, na);
  if (d < 8 || d % 8) return fail(SCE_ERR_INVALID, "similarity: d (%d) must be a positive multiple of 8", d);
  if (d > 8192) return fail(SCE_ERR_INVALID, "similarity: d = %d > 8192 is not supported by the row kernels", d);
  if ((a_normalize != 0 && a_normalize != 1) || (b && b_normalize != 0 && b_normalize != 1))
    return fail(SCE_ERR_INVALID, "similarity: a_normalize / b_normalize must be 0 or 1");
  const bool b_is_a = b == nullptr;
  if (!b_is_a && (mb < 1 || nb < 1)) return fail(SCE_ERR_INVALID, "similarity: mb (%d) and nb (%d) must be >= 1", mb, nb);
  const int Mb = b_is_a ? ma : mb, Nb = b_is_a ? na : nb;
  if (!pairs || n_pairs < 1) return fail(SCE_ERR_INVALID, "similarity: need at least one pair (pairs NULL or n_pairs = %d)", n_pairs);
  if (arith < SCE_ARITH_AUTO || arith > SCE_ARITH_F16F8) return fail(SCE_ERR_INVALID, "similarity: unknown arith %d", arith);
  if (arith == SCE_ARITH_F16F8 && d % 16)
    return fail(SCE_ERR_INVALID, "similarity: arith = F16F8 needs d (%d) to be a multiple of 16", d);
  if (!row_max && !col_max && !capacity) return fail(SCE_ERR_INVALID, "similarity: no output requested");
  if (capacity && !b_is_a) return fail(SCE_ERR_INVALID, "similarity: capacity is defined for self-pairs of one stack (b must be NULL)");
  const long long tiles = (long long)n_pairs * ((na + kBM - 1) / kBM) * ((Nb + kBN - 1) / kBN);
  if (tiles > 0x7FFFFFFFll) return fail(SCE_ERR_INVALID, "similarity: %lld tiles exceed the 32-bit tile index", tiles);
  std::vector<int> pv(pairs, pairs + 2 * (size_t)n_pairs);
  for (int q = 0; q < n_pairs; ++q)
    if (pv[2 * q] < 0 || pv[2 * q] >= ma || pv[2 * q + 1] < 0 || pv[2 * q + 1] >= Mb)
      return fail(SCE_ERR_INVALID, "similarity: pair %d = (%d, %d) outside [0, %d) x [0, %d)", q, pv[2 * q], pv[2 * q + 1], ma, Mb);
  std::vector<int> rows(ma + (b_is_a ? 0 : mb));
  for (int m = 0; m < ma; ++m) rows[m] = a_rows ? a_rows[m] : na;
  for (int m = 0; !b_is_a && m < mb; ++m) rows[ma + m] = b_rows ? b_rows[m] : nb;
  for (int m = 0; m < (int)rows.size(); ++m) {
    const int n = m < ma ? na : nb;
    if (rows[m] < 1 || rows[m] > n)
      return fail(SCE_ERR_INVALID, "similarity: rows[%d] of %s = %d outside [1, %d]", m < ma ? m : m - ma, m < ma ? "a" : "b", rows[m], n);
  }
  const size_t need = sim_workspace(ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr);
  if (int rc = check_workspace(workspace, workspace_bytes, need, "similarity: ")) return rc;

  // ---- device
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Launcher L{st};
  int dev = 0, sms = 0;
  if (int rc = query_device(&dev, &sms)) return rc;
  const SimOperand A{a, ma, na, a_normalize, a_norm_floor};
  const SimOperand B = b_is_a ? A : SimOperand{b, mb, nb, b_normalize, b_norm_floor};
  // AUTO: bf16x3. Unlike the training GEMMs, whose epilogues write operand planes and which are bound by the SM's data
  // paths, this GEMM's epilogue is light, and the widening of the E5M2 tiles made f16f8 the slower arithmetic here (H100,
  // config 2: 30.1 ms against 23.9 ms per pass) as well as the less accurate one (5e-6 against 1.3e-6 from fp64).
  // SCE_ARITH=f16f8 pins AUTO to f16f8 where d % 16 == 0. f16f8 splits a raw operand first and reads its range flag back
  // (one 4-byte copy + synchronise): a value fp16 cannot hold (|v| >= 65520 or NaN) moves a pinned AUTO to bf16x3 and
  // is an error under explicit F16F8.
  bool f8 = arith == SCE_ARITH_F16F8 || (arith == SCE_ARITH_AUTO && env_arith() == SCE_ARITH_F16F8 && d % 16 == 0);
  const bool raw = !A.normalize || (!b_is_a && !B.normalize);
  SimCarve w;
  if (f8 && raw) {
    sim_carve(static_cast<uint8_t*>(workspace), true, ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr, &w);
    CUDA_TRY(cudaMemsetAsync(w.flags, 0, kFlagWords * sizeof(uint32_t), st));
    int rc = SCE_OK;
    if (!A.normalize) rc = sim_planes<kArithF16F8>(L, A, d, w.a, w.flags);
    if (!rc && !b_is_a && !B.normalize) rc = sim_planes<kArithF16F8>(L, B, d, w.b, w.flags);
    if (rc) return rc;
    uint32_t bad = 0;
    CUDA_TRY(cudaMemcpyAsync(&bad, w.flags + kBadWord, sizeof(bad), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (bad) {
      if (arith == SCE_ARITH_F16F8)
        return fail(SCE_ERR_INVALID, "similarity: a raw operand holds a value fp16 cannot (|v| >= 65520 or NaN); use "
                                     "arith = BF16X3 or AUTO");
      f8 = false;
    }
  }
  sim_carve(static_cast<uint8_t*>(workspace), f8, ma, na, b_is_a ? 0 : mb, b_is_a ? 0 : nb, d, n_pairs, capacity != nullptr, &w);
  // the pair list and row counts are host locals: copies from pageable memory are staged before cudaMemcpyAsync returns
  CUDA_TRY(cudaMemcpyAsync(w.pairs, pv.data(), pv.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(w.a_rows, rows.data(), (size_t)ma * sizeof(int), cudaMemcpyHostToDevice, st));
  if (!b_is_a) CUDA_TRY(cudaMemcpyAsync(w.b_rows, rows.data() + ma, (size_t)mb * sizeof(int), cudaMemcpyHostToDevice, st));
  // (a raw operand split above for the range check is split again here: the planes of the arithmetic that runs)
  return f8 ? run_similarity_t<kArithF16F8>(L, A, B, b_is_a, d, n_pairs, w, row_max, col_max, capacity, dev, sms)
            : run_similarity_t<kArithBf16x3>(L, A, B, b_is_a, d, n_pairs, w, row_max, col_max, capacity, dev, sms);
}

}  // extern "C"
