// sce_abi.cu — libsce's per-thread error state, and the entry points that belong to no plan or pass: the version, the
// last error, the chunk row gather and the synthetic-data generator.
#include <cstdarg>
#include <cstdio>

#include "sce_engine.cuh"
#include "sce_synth.cuh"

static thread_local char g_err[512] = "";
int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

extern "C" {

int sce_version(void) { return SCE_VERSION; }
const char* sce_last_error(void) { return g_err; }

int sce_gather_rows(const void* chunk, int chunk_is_half, long long n_rows, int d, const long long* idx, int B,
                    const float* sub, float* out, void* stream) {
  if (!chunk || !out || B < 1 || d < 4 || d % 4) return fail(SCE_ERR_INVALID, "bad arguments to sce_gather_rows");
  Launcher L{static_cast<cudaStream_t>(stream)};
  const int blocks = (B + 7) / 8;
  if (chunk_is_half)
    return L.launch(gather_rows_kernel<__half>, blocks, 256, 0, static_cast<const __half*>(chunk), n_rows, d, idx, B, sub,
                    out);
  return L.launch(gather_rows_kernel<float>, blocks, 256, 0, static_cast<const float*>(chunk), n_rows, d, idx, B, sub, out);
}

int sce_synth_rows(const float* feats, int n_gt, int d, const float* probs, int group_rows, long long row0, int B,
                   unsigned long long seed, int zero_row_rule, float noise_scale, void* out, int out_half, int* row_nnz,
                   int* code_idx, float* code_val, int code_cap, void* stream) {
  // ---- arguments (all checked before any CUDA call)
  if (!feats || !probs || !out) return fail(SCE_ERR_INVALID, "synth_rows: feats, probs and out are required");
  if (n_gt < 1 || B < 1) return fail(SCE_ERR_INVALID, "synth_rows: n_gt (%d) and B (%d) must be >= 1", n_gt, B);
  if (d < 8 || d % 8) return fail(SCE_ERR_INVALID, "synth_rows: d (%d) must be a positive multiple of 8", d);
  if (d > 8192) return fail(SCE_ERR_INVALID, "synth_rows: d = %d > 8192 is not supported by the row kernels", d);
  if (group_rows < 1) return fail(SCE_ERR_INVALID, "synth_rows: group_rows (%d) must be >= 1", group_rows);
  if (row0 < 0) return fail(SCE_ERR_INVALID, "synth_rows: row0 (%lld) must be >= 0", row0);
  if ((zero_row_rule != 0 && zero_row_rule != 1) || (out_half != 0 && out_half != 1))
    return fail(SCE_ERR_INVALID, "synth_rows: zero_row_rule and out_half must be 0 or 1");
  if (!(noise_scale >= 0.f && noise_scale <= 3.0e38f))
    return fail(SCE_ERR_INVALID, "synth_rows: noise_scale must be finite and >= 0");
  if (!code_idx != !code_val) return fail(SCE_ERR_INVALID, "synth_rows: code_idx and code_val go together");
  if (code_idx && code_cap < 1) return fail(SCE_ERR_INVALID, "synth_rows: code_cap (%d) must be >= 1 with code lists", code_cap);
  if (reinterpret_cast<uintptr_t>(out) % 16 || reinterpret_cast<uintptr_t>(feats) % 16)
    return fail(SCE_ERR_INVALID, "synth_rows: out and feats must be 16-byte aligned");

  // ---- device
  SynthArgs a{feats, probs, n_gt, d, group_rows, B, row0, (uint32_t)seed, (uint32_t)(seed >> 32), zero_row_rule,
              noise_scale, out, out_half, row_nnz, code_idx, code_val, code_idx ? code_cap : 0};
  Launcher L{static_cast<cudaStream_t>(stream)};
  const unsigned rows8 = (unsigned)((B + 7) / 8);
  if (d <= 128) return L.launch(synth_rows_kernel<1, false>, rows8, 256, 0, a);
  if (d <= 256) return L.launch(synth_rows_kernel<2, false>, rows8, 256, 0, a);
  if (d <= 512) return L.launch(synth_rows_kernel<4, false>, rows8, 256, 0, a);
  if (d <= 1024) return L.launch(synth_rows_kernel<8, false>, rows8, 256, 0, a);
  return L.launch(synth_rows_kernel<8, true>, (unsigned)B, 32 * ((d + 1023) / 1024), 0, a);
}

}  // extern "C"
