//! Raw bindings of include/nb200.h.  Every function returns `nb200_status` (0 = OK) unless it returns a value directly.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_int, c_void};

macro_rules! opaque { ($($n:ident),*) => { $( #[repr(C)] pub struct $n { _p: [u8; 0] } )* } }
opaque!(nb200_ctx, nb200_cols, nb200_tree, nb200_channel, nb200_air, nb200_scheme);

pub const NB200_OK: c_int = 0;
pub const NB200_ERR_CUDA: c_int = 1;
pub const NB200_ERR_ARG: c_int = 2;
pub const NB200_ERR_NO_DEVICE: c_int = 3;
pub const NB200_ERR_OOM: c_int = 4;
pub const NB200_ERR_CONSTRAINTS: c_int = 5;
pub const NB200_ERR_STATE: c_int = 6;

#[repr(C)]
#[derive(Clone, Copy)]
pub struct nb200_sample_batch { pub point: [u32; 8], pub first_entry: usize, pub n_entries: usize }
#[repr(C)]
#[derive(Clone, Copy)]
pub struct nb200_sample_entry { pub column: u32, pub value: [u32; 4] }

extern "C" {
    // ---- context
    pub fn nb200_ctx_create(device: c_int, out: *mut *mut nb200_ctx) -> c_int;
    pub fn nb200_ctx_destroy(ctx: *mut nb200_ctx);
    pub fn nb200_last_error(ctx: *mut nb200_ctx) -> *const c_char;
    pub fn nb200_ctx_set_stream(ctx: *mut nb200_ctx, cuda_stream: *mut c_void) -> c_int;
    pub fn nb200_sync(ctx: *mut nb200_ctx) -> c_int;
    pub fn nb200_set_flavor(ctx: *mut nb200_ctx, merkle_hash: c_int, draw_domain_sep: c_int, pow_variant: c_int) -> c_int;
    pub fn nb200_launch_count(ctx: *mut nb200_ctx) -> u64;
    // ---- columns
    pub fn nb200_cols_alloc(ctx: *mut nb200_ctx, n_cols: usize, log_size: u32, out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_cols_from_device(ctx: *mut nb200_ctx, device_ptr: *mut c_void, n_cols: usize, log_size: u32, out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_cols_free(ctx: *mut nb200_ctx, cols: *mut nb200_cols);
    pub fn nb200_cols_count(cols: *const nb200_cols) -> usize;
    pub fn nb200_cols_log_size(cols: *const nb200_cols) -> u32;
    pub fn nb200_cols_device_ptr(cols: *const nb200_cols) -> *mut c_void;
    pub fn nb200_cols_upload(ctx: *mut nb200_ctx, cols: *mut nb200_cols, first: usize, n: usize, host: *const u32, coset_order: c_int) -> c_int;
    pub fn nb200_cols_download(ctx: *mut nb200_ctx, cols: *const nb200_cols, first: usize, n: usize, host: *mut u32) -> c_int;
    pub fn nb200_cols_finalize_order(ctx: *mut nb200_ctx, cols: *mut nb200_cols) -> c_int;
    // ---- PolyOps
    pub fn nb200_twiddles_prepare(ctx: *mut nb200_ctx, max_domain_log: u32) -> c_int;
    pub fn nb200_twiddles_domain_log(ctx: *mut nb200_ctx) -> u32;
    pub fn nb200_twiddles_download(ctx: *mut nb200_ctx, tw: *mut u32, itw: *mut u32) -> c_int;
    pub fn nb200_interpolate(ctx: *mut nb200_ctx, cols: *mut nb200_cols) -> c_int;
    pub fn nb200_evaluate(ctx: *mut nb200_ctx, coeffs: *const nb200_cols, log_blowup: u32, out: *mut nb200_cols) -> c_int;
    pub fn nb200_interpolate_evaluate(ctx: *mut nb200_ctx, evals: *const nb200_cols, log_blowup: u32, coeffs: *mut nb200_cols, lde: *mut nb200_cols) -> c_int;
    pub fn nb200_eval_at_points(ctx: *mut nb200_ctx, coeffs: *const nb200_cols, points_xy: *const u32, n_points: usize, out_qm31: *mut u32) -> c_int;
    // ---- MerkleOps
    pub fn nb200_merkle_commit(ctx: *mut nb200_ctx, batches: *const *const nb200_cols, n_batches: usize, out: *mut *mut nb200_tree, root: *mut u8) -> c_int;
    pub fn nb200_tree_free(ctx: *mut nb200_ctx, tree: *mut nb200_tree);
    pub fn nb200_tree_log_size(tree: *const nb200_tree) -> u32;
    pub fn nb200_tree_layer_download(ctx: *mut nb200_ctx, tree: *const nb200_tree, layer_log: u32, out: *mut u8) -> c_int;
    pub fn nb200_merkle_decommit(ctx: *mut nb200_ctx, tree: *const nb200_tree, batches: *const *const nb200_cols, n_batches: usize,
                                 q_log_sizes: *const u32, q_counts: *const u64, q_positions: *const u64, n_sizes: usize,
                                 queried_values: *mut *mut u32, n_queried: *mut usize, hash_witness: *mut *mut u8, n_hashes: *mut usize,
                                 column_witness: *mut *mut u32, n_column_witness: *mut usize) -> c_int;
    pub fn nb200_merkle_decommit_plan(max_log: u32, col_log_sizes: *const u32, n_cols: usize,
                                      q_log_sizes: *const u32, q_counts: *const u64, q_positions: *const u64, n_sizes: usize,
                                      values: *mut *mut u64, n_values: *mut usize, hashes: *mut *mut u64, n_hashes: *mut usize) -> c_int;
    pub fn nb200_free(p: *mut c_void);
    pub fn nb200_hash_node(merkle_hash: c_int, left: *const u8, right: *const u8, values: *const u32, n_values: usize, out: *mut u8) -> c_int;
    // ---- fused commitment
    pub fn nb200_commit_evals(ctx: *mut nb200_ctx, eval_batches: *const *const nb200_cols, n_batches: usize, log_blowup: u32,
                              coeffs_io: *mut *mut nb200_cols, lde_io: *mut *mut nb200_cols, tree_out: *mut *mut nb200_tree, root: *mut u8) -> c_int;
    pub fn nb200_host_alloc(bytes: usize, out: *mut *mut c_void) -> c_int;
    pub fn nb200_host_free(p: *mut c_void);
    pub fn nb200_commit_host(ctx: *mut nb200_ctx, host_batches: *const *const u32, n_cols: *const usize, log_sizes: *const u32, n_batches: usize,
                             coset_order: c_int, log_blowup: u32, evals_io: *mut *mut nb200_cols, coeffs_io: *mut *mut nb200_cols,
                             lde_io: *mut *mut nb200_cols, tree_out: *mut *mut nb200_tree, root: *mut u8) -> c_int;
    pub fn nb200_commit_host_packed(ctx: *mut nb200_ctx, host_batches: *const *const c_void, elem_bytes: *const u32, n_cols: *const usize,
                                    log_sizes: *const u32, n_batches: usize, coset_order: c_int, log_blowup: u32, evals_io: *mut *mut nb200_cols,
                                    coeffs_io: *mut *mut nb200_cols, lde_io: *mut *mut nb200_cols, tree_out: *mut *mut nb200_tree, root: *mut u8) -> c_int;
    // ---- the keccak extension's main trace filled on the device from its side note (out: 5 batches)
    pub fn nb200_keccak_main_trace(ctx: *mut nb200_ctx, n_perms: usize, inputs: *const u64, addresses: *const u32, timestamps: *const u32,
                                   out: *mut *mut nb200_cols) -> c_int;
    // ---- RamInitFinal's main trace filled on the device from the keccak side note and the public initial memory (out: caller's 10-column batch)
    pub fn nb200_ram_init_final_trace(ctx: *mut nb200_ctx, n_perms: usize, inputs: *const u64, addresses: *const u32, timestamps: *const u32,
                                      n_init: usize, init_addresses: *const u32, init_values: *const u8, log_size: u32, out: *mut nb200_cols,
                                      n_rows_out: *mut usize) -> c_int;
    // ---- the v1 main component's main trace filled on the device from an ADD / ADDI program's step record (out: caller's 347-column batch)
    pub fn nb200_v1_main_trace(ctx: *mut nb200_ctx, n_steps: usize, steps: *const u32, n_prog: usize, final_ctr: *const u32, log_size: u32,
                               out: *mut nb200_cols) -> c_int;
    // ---- the same fill for a program of RV32I's ALU instructions, ADD ... SRAI (out: caller's 347-column batch)
    pub fn nb200_v1_alu_trace(ctx: *mut nb200_ctx, n_steps: usize, steps: *const u32, n_prog: usize, final_ctr: *const u32, log_size: u32,
                              out: *mut nb200_cols) -> c_int;
    // ---- the same fill for a looping program of those, RV32I's branches, JAL, JALR, LUI and AUIPC (out: caller's 347-column batch)
    pub fn nb200_v1_control_trace(ctx: *mut nb200_ctx, n_steps: usize, steps: *const u32, n_prog: usize, final_ctr: *const u32, log_size: u32,
                                  out: *mut nb200_cols) -> c_int;
    // ---- one commitment over N GPUs (NCCL inside the library)
    pub fn nb200_comm_unique_id_bytes() -> usize;
    pub fn nb200_comm_get_unique_id(id_out: *mut u8) -> c_int;
    pub fn nb200_comm_init(ctx: *mut nb200_ctx, rank: c_int, world: c_int, unique_id: *const u8) -> c_int;
    pub fn nb200_comm_destroy(ctx: *mut nb200_ctx);
    pub fn nb200_comm_rank(ctx: *const nb200_ctx) -> c_int;
    pub fn nb200_comm_world(ctx: *const nb200_ctx) -> c_int;
    pub fn nb200_shard_range(total_cols: usize, world: c_int, rank: c_int, first: *mut usize, count: *mut usize) -> c_int;
    pub fn nb200_comm_all_gather(ctx: *mut nb200_ctx, mine: *const u8, bytes: usize, out: *mut u8) -> c_int;
    pub fn nb200_commit_sharded(ctx: *mut nb200_ctx, shard_evals: *const nb200_cols, total_cols: usize, log_size: u32, log_blowup: u32,
                                replicated: *const *const nb200_cols, n_replicated: usize, coeffs_out: *mut *mut nb200_cols, rows_out: *mut *mut nb200_cols,
                                subtree_out: *mut *mut nb200_tree, caps_out: *mut u8, root: *mut u8) -> c_int;
    pub fn nb200_scheme_commit_sharded(s: *mut nb200_scheme, big_shard: *const nb200_cols, total_big: usize, log_size: u32, small: *const *const nb200_cols, n_small: usize,
                                       replicate_cols: *const u32, n_replicate: usize, keep_eval_rows: c_int, ch: *mut nb200_channel, root: *mut u8) -> c_int;
    pub fn nb200_gen_interaction_trace_sharded(s: *mut nb200_scheme, air: *const nb200_air, component: u32, params: *const u32, n_params: usize,
                                               shard_out: *mut *mut nb200_cols, claimed_sum: *mut u32) -> c_int;
    // ---- Blake2sChannel
    pub fn nb200_channel_new(ctx: *mut nb200_ctx, out: *mut *mut nb200_channel) -> c_int;
    pub fn nb200_channel_clone(ch: *const nb200_channel, out: *mut *mut nb200_channel) -> c_int;
    pub fn nb200_channel_free(ch: *mut nb200_channel);
    pub fn nb200_channel_digest(ch: *const nb200_channel, out: *mut u8);
    pub fn nb200_channel_mix_u64(ch: *mut nb200_channel, v: u64);
    pub fn nb200_channel_mix_u32s(ch: *mut nb200_channel, words: *const u32, n: usize);
    pub fn nb200_channel_mix_felts(ch: *mut nb200_channel, qm31s: *const u32, n: usize);
    pub fn nb200_channel_mix_root(ch: *mut nb200_channel, root: *const u8);
    pub fn nb200_channel_draw_felt(ch: *mut nb200_channel, out: *mut u32);
    pub fn nb200_channel_draw_felts(ch: *mut nb200_channel, n: usize, out: *mut u32);
    pub fn nb200_channel_draw_random_bytes(ch: *mut nb200_channel, out: *mut u8);
    pub fn nb200_device_channel_draw(ctx: *mut nb200_ctx, digest: *const u8, n_sent: u64, roots: *const u8, n: usize,
                                     felts_out: *mut u32, digest_out: *mut u8, n_sent_out: *mut u64) -> c_int;
    // ---- AIR
    pub fn nb200_air_load(ctx: *mut nb200_ctx, words: *const u32, n_words: usize, out: *mut *mut nb200_air) -> c_int;
    pub fn nb200_air_free(air: *mut nb200_air);
    pub fn nb200_air_n_params(air: *const nb200_air) -> u32;
    pub fn nb200_air_n_components(air: *const nb200_air) -> u32;
    pub fn nb200_air_n_constraints(air: *const nb200_air, component: u32) -> u32;
    pub fn nb200_air_kernel_source(air: *const nb200_air, component: u32, which: c_int, out: *mut *mut c_char) -> c_int;
    pub fn nb200_kernel_source_key(source: *const c_char) -> u64;
    pub fn nb200_air_constraint_degrees(air: *const nb200_air, component: u32, degrees: *mut u32, n: usize) -> c_int;
    pub fn nb200_air_d2_masks(air: *const nb200_air, component: u32, flags: *mut u8, n: usize) -> c_int;
    pub fn nb200_air_max_log_expand(air: *const nb200_air) -> u32;
    // ---- CommitmentSchemeProver / prove
    pub fn nb200_scheme_new(ctx: *mut nb200_ctx, pow_bits: u32, log_blowup: u32, log_last_layer_degree_bound: u32, n_queries: u32, out: *mut *mut nb200_scheme) -> c_int;
    pub fn nb200_scheme_free(s: *mut nb200_scheme);
    pub fn nb200_scheme_set_constraint_log_degree(s: *mut nb200_scheme, log_expand: u32) -> c_int;
    pub fn nb200_scheme_commit(s: *mut nb200_scheme, eval_batches: *const *const nb200_cols, n_batches: usize, ch: *mut nb200_channel, root: *mut u8) -> c_int;
    pub fn nb200_scheme_commit_host(s: *mut nb200_scheme, host_batches: *const *const u32, n_cols: *const usize, log_sizes: *const u32, n_batches: usize,
                                    coset_order: c_int, ch: *mut nb200_channel, root: *mut u8, evals_out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_scheme_commit_host_packed(s: *mut nb200_scheme, host_batches: *const *const c_void, elem_bytes: *const u32, n_cols: *const usize,
                                           log_sizes: *const u32, n_batches: usize, coset_order: c_int, ch: *mut nb200_channel, root: *mut u8,
                                           evals_out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_gen_interaction_trace(ctx: *mut nb200_ctx, air: *const nb200_air, component: u32, tree0: *const *const nb200_cols, n0: usize,
                                       tree1: *const *const nb200_cols, n1: usize, params: *const u32, n_params: usize,
                                       out: *mut *mut nb200_cols, claimed_sum: *mut u32) -> c_int;
    pub fn nb200_prove(s: *mut nb200_scheme, air: *const nb200_air, params: *const u32, n_params: usize, ch: *mut nb200_channel,
                       proof_out: *mut *mut u8, proof_len: *mut usize) -> c_int;
    pub fn nb200_check_constraints(ctx: *mut nb200_ctx, air: *const nb200_air, component: u32, tree0: *const *const nb200_cols, n0: usize,
                                   tree1: *const *const nb200_cols, n1: usize, tree2: *const *const nb200_cols, n2: usize,
                                   params: *const u32, n_params: usize, n_failing: *mut u64, first_row: *mut u64, n: usize) -> c_int;
    // ---- lookup-table multiplicities counted on the device from the AIR's lookups
    pub fn nb200_air_lookup_tables(air: *const nb200_air, component: u32, kind: *mut u32, relation: *mut u32, arg: *mut u32, n: usize) -> c_int;
    pub fn nb200_air_count_kernel_source(air: *const nb200_air, component: u32, out: *mut *mut c_char) -> c_int;
    pub fn nb200_table_multiplicities(ctx: *mut nb200_ctx, air: *const nb200_air, tree0: *const *const nb200_cols, n0: usize,
                                      tree1: *const *mut nb200_cols, n1: usize, n_unmatched: *mut u64, first_unmatched: *mut u32) -> c_int;
    pub fn nb200_table_multiplicities_first_row(ctx: *mut nb200_ctx, air: *const nb200_air, tree0: *const *const nb200_cols, n0: usize,
                                                tree1: *const *mut nb200_cols, n1: usize, n_unmatched: *mut u64, first_unmatched: *mut u32,
                                                n_repeated: *mut u64) -> c_int;
    // ---- backend-trait level operations
    pub fn nb200_constraint_quotients(s: *mut nb200_scheme, air: *const nb200_air, component: u32, params: *const u32, n_params: usize,
                                      coeffs: *const u32, n_coeffs: usize, accum: *mut nb200_cols) -> c_int;
    pub fn nb200_constraint_quotients_half(s: *mut nb200_scheme, air: *const nb200_air, component: u32, params: *const u32, n_params: usize,
                                           coeffs: *const u32, n_coeffs: usize, q_d1: *mut nb200_cols, q_high_d2: *mut nb200_cols,
                                           q_high_d1: *mut nb200_cols) -> c_int;
    pub fn nb200_accumulate(ctx: *mut nb200_ctx, a: *mut nb200_cols, b: *const nb200_cols) -> c_int;
    pub fn nb200_fri_quotients(ctx: *mut nb200_ctx, batches: *const *const nb200_cols, n_batches: usize, log_size: u32,
                               sample_batches: *const nb200_sample_batch, n_sample_batches: usize, entries: *const nb200_sample_entry, n_entries: usize,
                               random_coeff: *const u32, out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_fri_quotients_from_coeffs(ctx: *mut nb200_ctx, coeffs: *const *const nb200_cols, n_batches: usize, log_size: u32, log_blowup: u32,
                                           sample_batches: *const nb200_sample_batch, n_sample_batches: usize, entries: *const nb200_sample_entry,
                                           n_entries: usize, random_coeff: *const u32, out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_deep_plan(sample_batches: *const nb200_sample_batch, n_sample_batches: usize, entries: *const nb200_sample_entry, n_entries: usize,
                           random_coeff: *const u32, lines_out: *mut u32, alphas_out: *mut u32) -> c_int;
    pub fn nb200_fold_circle_into_line(ctx: *mut nb200_ctx, dst: *mut nb200_cols, src: *const nb200_cols, alpha: *const u32) -> c_int;
    pub fn nb200_fold_line(ctx: *mut nb200_ctx, src: *const nb200_cols, alpha: *const u32, dst_out: *mut *mut nb200_cols) -> c_int;
    pub fn nb200_grind(ctx: *mut nb200_ctx, digest: *const u8, pow_bits: u32, nonce_out: *mut u64) -> c_int;
}
