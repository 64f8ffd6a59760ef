//! Owning wrappers over the C ABI.  One `Context` = one GPU + one proving thread (the reference drives the protocol from a
//! single thread too: prover/src/machine.rs:130-297; tests are #[serial]).
use std::ffi::CStr;
use std::os::raw::c_void;
use std::ptr;
use std::rc::Rc;

use stwo::core::fields::qm31::SecureField;
use stwo::core::fields::m31::BaseField;

use crate::ffi::*;

#[derive(Debug, thiserror::Error)]
pub enum Error {
    #[error("no CUDA device: libnexus_b200 has no CPU fallback ({0})")]
    NoDevice(String),
    /// `ProvingError::ConstraintsNotSatisfied` (prover/src/lib.rs:24-31)
    #[error("constraints not satisfied")]
    ConstraintsNotSatisfied,
    #[error("nb200 status {status}: {message}")]
    Backend { status: i32, message: String },
}
pub type Result<T> = std::result::Result<T, Error>;

struct CtxHandle(*mut nb200_ctx);
impl Drop for CtxHandle {
    fn drop(&mut self) { unsafe { nb200_ctx_destroy(self.0) } }
}

/// One GPU: device, stream, twiddle cache (`CommitmentSchemeProver::new(config, &twiddles)` ownership lives here).
#[derive(Clone)]
pub struct Context(Rc<CtxHandle>);

fn secure_to_words(v: &[SecureField]) -> Vec<u32> {
    v.iter().flat_map(|q| q.to_m31_array().map(|m: BaseField| m.0)).collect()
}
fn words_to_secure(w: &[u32]) -> SecureField {
    SecureField::from_m31_array([BaseField::from_u32_unchecked(w[0]), BaseField::from_u32_unchecked(w[1]),
                                 BaseField::from_u32_unchecked(w[2]), BaseField::from_u32_unchecked(w[3])])
}

impl Context {
    pub fn new(device: i32) -> Result<Self> {
        let mut h = ptr::null_mut();
        let st = unsafe { nb200_ctx_create(device, &mut h) };
        if st != NB200_OK {
            let msg = unsafe { CStr::from_ptr(nb200_last_error(ptr::null_mut())) }.to_string_lossy().into_owned();
            return Err(if st == NB200_ERR_NO_DEVICE { Error::NoDevice(msg) } else { Error::Backend { status: st, message: msg } });
        }
        Ok(Context(Rc::new(CtxHandle(h))))
    }
    pub(crate) fn raw(&self) -> *mut nb200_ctx { self.0 .0 }
    pub(crate) fn check(&self, st: i32) -> Result<()> {
        match st {
            NB200_OK => Ok(()),
            NB200_ERR_CONSTRAINTS => Err(Error::ConstraintsNotSatisfied),
            _ => Err(Error::Backend { status: st, message: unsafe { CStr::from_ptr(nb200_last_error(self.raw())) }.to_string_lossy().into_owned() }),
        }
    }
    /// transcript-affecting variants (DESIGN.md "parity risk switches"); the differential test flips them when a root or a draw differs
    pub fn set_flavor(&self, merkle_hash: i32, draw_domain_sep: i32) -> Result<()> {
        self.check(unsafe { nb200_set_flavor(self.raw(), merkle_hash, draw_domain_sep, 0) })
    }
    /// `SimdBackend::precompute_twiddles(CanonicCoset::new(max_domain_log).circle_domain().half_coset)` — machine.rs:186-194
    pub fn precompute_twiddles(&self, max_domain_log: u32) -> Result<()> {
        self.check(unsafe { nb200_twiddles_prepare(self.raw(), max_domain_log) })
    }
    /// Upload host columns of one log size (trace/coset order; the device applies `finalize_columns`,
    /// prover/src/trace/utils.rs:94-106) as one batch.  `cols` are `&[BaseField]` slices reinterpreted as u32 words.
    pub fn upload_coset_order(&self, cols: &[&[BaseField]], log_size: u32) -> Result<Columns> { self.upload(cols, log_size, true) }
    /// columns that are already in bit-reversed circle-domain order (`TracesBuilder::finalize`, `BaseColumn::as_slice`)
    pub fn upload_finalized(&self, cols: &[&[BaseField]], log_size: u32) -> Result<Columns> { self.upload(cols, log_size, false) }
    fn upload(&self, cols: &[&[BaseField]], log_size: u32, coset_order: bool) -> Result<Columns> {
        let mut h = ptr::null_mut();
        self.check(unsafe { nb200_cols_alloc(self.raw(), cols.len(), log_size, &mut h) })?;
        let out = Columns { ctx: self.clone(), h };
        for (i, c) in cols.iter().enumerate() {
            assert_eq!(c.len(), 1usize << log_size);
            // BaseField is #[repr(transparent)] over u32 (stwo core/fields/m31.rs)
            self.check(unsafe { nb200_cols_upload(self.raw(), h, i, 1, c.as_ptr() as *const u32, coset_order as i32) })?;
        }
        Ok(out)
    }
    /// NCCL communicator of this context (one process per GPU): rank 0 calls `comm_unique_id()`, ships the bytes to the other ranks, all call `comm_init`.
    pub fn comm_unique_id() -> Result<Vec<u8>> {
        let mut id = vec![0u8; unsafe { nb200_comm_unique_id_bytes() }];
        let st = unsafe { nb200_comm_get_unique_id(id.as_mut_ptr()) };
        if st != NB200_OK { return Err(Error::Backend { status: st, message: "nb200_comm_get_unique_id failed (is libnccl loadable?)".into() }); }
        Ok(id)
    }
    pub fn comm_init(&self, rank: i32, world: i32, unique_id: &[u8]) -> Result<()> {
        self.check(unsafe { nb200_comm_init(self.raw(), rank, world, unique_id.as_ptr()) })
    }
    /// the 16-column-aligned column range rank `rank` of `world` transforms (`nb200_shard_range`)
    pub fn shard_range(total_cols: usize, world: i32, rank: i32) -> (usize, usize) {
        let (mut f, mut c) = (0usize, 0usize);
        unsafe { nb200_shard_range(total_cols, world, rank, &mut f, &mut c) };
        (f, c)
    }
    pub fn channel(&self) -> Result<Channel> {
        let mut h = ptr::null_mut();
        self.check(unsafe { nb200_channel_new(self.raw(), &mut h) })?;
        Ok(Channel { h })
    }
    pub fn scheme(&self, p: PcsParams) -> Result<Scheme> {
        let mut h = ptr::null_mut();
        self.check(unsafe { nb200_scheme_new(self.raw(), p.pow_bits, p.log_blowup_factor, p.log_last_layer_degree_bound, p.n_queries, &mut h) })?;
        Ok(Scheme { ctx: self.clone(), h })
    }
    pub fn air(&self, words: &[u32]) -> Result<Air> {
        let mut h = ptr::null_mut();
        self.check(unsafe { nb200_air_load(self.raw(), words.as_ptr(), words.len(), &mut h) })?;
        Ok(Air { h })
    }
    /// `generate_interaction_trace` of one component on the device (machine.rs:242-260, LogupTraceGenerator semantics)
    pub fn gen_interaction_trace(&self, air: &Air, component: u32, tree0: &[&Columns], tree1: &[&Columns], params: &[SecureField])
        -> Result<(Columns, SecureField)> {
        let t0: Vec<*const nb200_cols> = tree0.iter().map(|c| c.h as *const _).collect();
        let t1: Vec<*const nb200_cols> = tree1.iter().map(|c| c.h as *const _).collect();
        let p = secure_to_words(params);
        let (mut out, mut cs) = (ptr::null_mut(), [0u32; 4]);
        self.check(unsafe { nb200_gen_interaction_trace(self.raw(), air.h, component, t0.as_ptr(), t0.len(), t1.as_ptr(), t1.len(),
                                                        p.as_ptr(), params.len(), &mut out, cs.as_mut_ptr()) })?;
        Ok((Columns { ctx: self.clone(), h: out }, words_to_secure(&cs)))
    }
    /// `assert_constraints_on_polys` of one component on the device: for every constraint that fails somewhere,
    /// `(constraint index, failing rows, first failing row in trace order)`.  An empty vector: every constraint holds on every row.
    pub fn check_constraints(&self, air: &Air, component: u32, tree0: &[&Columns], tree1: &[&Columns], tree2: &[&Columns], params: &[SecureField])
        -> Result<Vec<(usize, u64, u64)>> {
        let t: Vec<Vec<*const nb200_cols>> = [tree0, tree1, tree2].iter().map(|tr| tr.iter().map(|c| c.h as *const _).collect()).collect();
        let n = unsafe { nb200_air_n_constraints(air.h, component) } as usize;
        let p = secure_to_words(params);
        let (mut failing, mut first) = (vec![0u64; n], vec![0u64; n]);
        self.check(unsafe { nb200_check_constraints(self.raw(), air.h, component, t[0].as_ptr(), t[0].len(), t[1].as_ptr(), t[1].len(),
                                                    t[2].as_ptr(), t[2].len(), p.as_ptr(), params.len(), failing.as_mut_ptr(), first.as_mut_ptr(), n) })?;
        Ok((0..n).filter(|&k| failing[k] != 0).map(|k| (k, failing[k], first[k])).collect())
    }
}

/// `PcsConfig { pow_bits, fri_config: FriConfig { log_blowup_factor, log_last_layer_degree_bound, n_queries } }`
#[derive(Clone, Copy, Debug)]
pub struct PcsParams { pub pow_bits: u32, pub log_blowup_factor: u32, pub log_last_layer_degree_bound: u32, pub n_queries: u32 }
impl From<stwo::core::pcs::PcsConfig> for PcsParams {
    fn from(c: stwo::core::pcs::PcsConfig) -> Self {
        PcsParams { pow_bits: c.pow_bits, log_blowup_factor: c.fri_config.log_blowup_factor,
                    log_last_layer_degree_bound: c.fri_config.log_last_layer_degree_bound, n_queries: c.fri_config.n_queries as u32 }
    }
}

/// A batch of device columns of one log size (the hand-off type that replaces `Vec<CircleEvaluation<SimdBackend, ..>>`).
pub struct Columns { ctx: Context, pub(crate) h: *mut nb200_cols }
impl Drop for Columns { fn drop(&mut self) { unsafe { nb200_cols_free(self.ctx.raw(), self.h) } } }
impl Columns {
    pub fn n_cols(&self) -> usize { unsafe { nb200_cols_count(self.h) } }
    pub fn log_size(&self) -> u32 { unsafe { nb200_cols_log_size(self.h) } }
}

/// `Blake2sChannel` (the library owns the implementation so that the coarse `prove` and this shim share one transcript)
pub struct Channel { pub(crate) h: *mut nb200_channel }
impl Drop for Channel { fn drop(&mut self) { unsafe { nb200_channel_free(self.h) } } }
impl Channel {
    pub fn mix_u64(&mut self, v: u64) { unsafe { nb200_channel_mix_u64(self.h, v) } }
    pub fn mix_felts(&mut self, felts: &[SecureField]) { let w = secure_to_words(felts); unsafe { nb200_channel_mix_felts(self.h, w.as_ptr(), felts.len()) } }
    pub fn draw_felts(&mut self, n: usize) -> Vec<SecureField> {
        let mut w = vec![0u32; 4 * n];
        unsafe { nb200_channel_draw_felts(self.h, n, w.as_mut_ptr()) };
        w.chunks(4).map(words_to_secure).collect()
    }
    pub fn digest(&self) -> [u8; 32] { let mut d = [0u8; 32]; unsafe { nb200_channel_digest(self.h, d.as_mut_ptr()) }; d }
}

pub struct Air { pub(crate) h: *mut nb200_air }
impl Drop for Air { fn drop(&mut self) { unsafe { nb200_air_free(self.h) } } }
impl Air {
    pub fn n_components(&self) -> u32 { unsafe { nb200_air_n_components(self.h) } }
    pub fn max_log_expand(&self) -> u32 { unsafe { nb200_air_max_log_expand(self.h) } }
}

/// `CommitmentSchemeProver::<CudaBackend, Blake2sMerkleChannel>`
pub struct Scheme { ctx: Context, h: *mut nb200_scheme }
impl Drop for Scheme { fn drop(&mut self) { unsafe { nb200_scheme_free(self.h) } } }
impl Scheme {
    pub fn set_constraint_log_degree(&self, log_expand: u32) -> Result<()> {
        self.ctx.check(unsafe { nb200_scheme_set_constraint_log_degree(self.h, log_expand) })
    }
    /// `tree_builder.extend_evals(batches..); tree_builder.commit(channel)` — machine.rs:208-263.  Returns the root.
    pub fn commit(&mut self, batches: &[&Columns], ch: &mut Channel) -> Result<[u8; 32]> {
        let b: Vec<*const nb200_cols> = batches.iter().map(|c| c.h as *const _).collect();
        let mut root = [0u8; 32];
        self.ctx.check(unsafe { nb200_scheme_commit(self.h, b.as_ptr(), b.len(), ch.h, root.as_mut_ptr()) })?;
        Ok(root)
    }
    /// One proof over N GPUs: the tree's leading `total_big` columns of 2^log_size rows (the main component's) are sharded — `big_shard` is this rank's
    /// `shard_range` of them — and the smaller batches are replicated; `replicate_cols` lists the big columns the AIR reads at a row offset.
    /// Call on every rank with the same arguments (DESIGN.md §5); returns the root of the WHOLE tree.
    pub fn commit_sharded(&mut self, big_shard: Option<&Columns>, total_big: usize, log_size: u32, small: &[&Columns], replicate_cols: &[u32],
                          keep_eval_rows: bool, ch: &mut Channel) -> Result<[u8; 32]> {
        let b: Vec<*const nb200_cols> = small.iter().map(|c| c.h as *const _).collect();
        let mut root = [0u8; 32];
        self.ctx.check(unsafe { nb200_scheme_commit_sharded(self.h, big_shard.map_or(ptr::null(), |c| c.h as *const _), total_big, log_size, b.as_ptr(), b.len(),
                                                            replicate_cols.as_ptr(), replicate_cols.len(), keep_eval_rows as i32, ch.h, root.as_mut_ptr()) })?;
        Ok(root)
    }
    /// LogUp interaction trace of the sharded (main) component from the trace rows kept by `commit_sharded(.., keep_eval_rows = true, ..)`:
    /// returns this rank's COLUMN shard of the 4 x n_logup_cols interaction columns and the component's claimed sum (same on every rank).
    pub fn gen_interaction_trace_sharded(&self, air: &Air, component: u32, params: &[SecureField]) -> Result<(Columns, SecureField)> {
        let p = secure_to_words(params);
        let (mut out, mut cs) = (ptr::null_mut(), [0u32; 4]);
        self.ctx.check(unsafe { nb200_gen_interaction_trace_sharded(self.h, air.h, component, p.as_ptr(), params.len(), &mut out, cs.as_mut_ptr()) })?;
        Ok((Columns { ctx: self.ctx.clone(), h: out }, words_to_secure(&cs)))
    }
    /// `stwo::prover::prove::<B, Blake2sMerkleChannel>(components, channel, commitment_scheme)` — machine.rs:286-290.
    /// Returns `postcard(StarkProof<Blake2sMerkleHasher>)`.
    pub fn prove(self, air: &Air, params: &[SecureField], ch: &mut Channel) -> Result<Vec<u8>> {
        let p = secure_to_words(params);
        let (mut out, mut len) = (ptr::null_mut::<u8>(), 0usize);
        self.ctx.check(unsafe { nb200_prove(self.h, air.h, p.as_ptr(), params.len(), ch.h, &mut out, &mut len) })?;
        let bytes = unsafe { std::slice::from_raw_parts(out, len) }.to_vec();
        unsafe { nb200_free(out as *mut c_void) };
        Ok(bytes)
    }
}
