// Test harness (not product): the gunzip passes of brpc_b200/csrc/b2_h2.cuh — k_h2_set_gunzip, k_h2_gz_select, k_h2_gz_size, k_h2_gz_place,
// k_h2_gz_inflate — built for the host on top of the client harness (h2_client_host.cc), launched after k_h2_client_consume the way
// brpc_b200/csrc/b2_api.cu launches them: one "thread" per run or per descriptor slot, in the same order.
#include "h2_client_host.cc"

extern "C" {
void h2g_set_gunzip(h2h_ctx* c, uint32_t conn, int enable) { blockDim.x = 1; blockIdx.x = 0; threadIdx.x = 0; k_h2_set_gunzip(c->conns, conn, enable); }
// b2_h2_client_process_batch with the passes: gz holds n_runs * per_run_calls words, merge_scratch n_runs * B2_H2_HEADER_BYTES
void h2g_consume(h2h_ctx* c, const uint8_t* bytes, const b2_run* runs, uint32_t n_runs, b2_h2_run_status* rs, b2_h2_call* calls,
                 uint32_t per_run_calls, uint8_t* out, uint32_t region, uint8_t* merge_scratch, uint32_t* gz) {
    h2c_consume(c, bytes, runs, n_runs, rs, calls, per_run_calls, out, region);
    blockDim.x = 1; threadIdx.x = 0;
    for (uint32_t r = 0; r < n_runs; r++) { blockIdx.x = r; k_h2_gz_select<b2_h2_call>(bytes, runs, n_runs, c->conns, rs, calls, per_run_calls, out, merge_scratch, gz); }
    for (uint32_t t = 0; t < n_runs * per_run_calls; t++) { blockIdx.x = t; k_h2_gz_size<b2_h2_call>(bytes, n_runs, rs, calls, per_run_calls, out, gz); }
    for (uint32_t r = 0; r < n_runs; r++) { blockIdx.x = r; k_h2_gz_place<b2_h2_call>(n_runs, rs, calls, per_run_calls, region, gz); }
    for (uint32_t t = 0; t < n_runs * per_run_calls; t++) { blockIdx.x = t; k_h2_gz_inflate<b2_h2_call>(bytes, n_runs, rs, calls, per_run_calls, out, gz); }
}
}
