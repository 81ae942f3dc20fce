//! `ark-groth16-b200`: ark-groth16 0.5's prover API on top of `libg16b200.so` (H100 / sm_90a CUDA kernels).
//!
//! What is replaced (file:line of arkworks-rs/groth16 @ d570ee5):
//!   * `Groth16::<E>::create_proof_with_reduction_and_matrices`   src/prover.rs:26-51   -> [`B200Prover::create_proof_with_reduction_and_matrices`]
//!   * `Groth16::<E>::create_proof_with_reduction` / `_no_zk` / `create_random_proof_with_reduction`
//!                                                                  src/prover.rs:138-204 -> methods of the same names
//!   * `impl SNARK for Groth16<E, QAP>`                             src/lib.rs:59-97      -> [`Groth16B200`] (setup / verify forwarded)
//!   * `R1CSToQAP::witness_map_from_matrices`                       src/r1cs_to_qap.rs:172-235 -> [`GpuReduction`] (NTT path only,
//!     selectable as `ark_groth16::Groth16<E, GpuReduction>` without touching the MSMs)
//! The MSMs have no hook inside ark-groth16 (src/prover.rs:66,74,262 call `msm_bigint` on `E::G1` / `E::G2` directly),
//! hence the sibling prover type instead of a trait implementation.
//!
//! Memory image (include/g16b200.h): a field element is its `[u64; N]` Montgomery limbs exactly as `ark_ff::Fp` stores them
//! (`Fp(pub BigInt<N>, PhantomData)`), so slices of scalars cross the ABI by pointer; affine points are repacked to
//! `x || y` (G2: `x.c0 || x.c1 || y.c0 || y.c1`) with all-zero limbs for the point at infinity, because
//! `short_weierstrass::Affine { x, y, infinity }` is not `repr(C)`.
//!
//! This crate is SOURCE ONLY in the repository that carries the CUDA library (no Rust toolchain in its build image); the
//! same C symbols are exercised by the Python binding in every test.  `tests/test_shim_abi.py` keeps `sys.rs` in step with
//! the header.

pub mod sys;

use ark_crypto_primitives::snark::{CircuitSpecificSetupSNARK, SNARK};
use ark_ec::{
    pairing::Pairing,
    short_weierstrass::{Affine, SWCurveConfig},
    AffineRepr,
};
use ark_ff::{Field, PrimeField, UniformRand, Zero};
use ark_groth16::{
    r1cs_to_qap::{LibsnarkReduction, R1CSToQAP},
    Groth16, PreparedVerifyingKey, Proof, ProvingKey, VerifyingKey,
};
use ark_poly::EvaluationDomain;
use ark_relations::r1cs::{
    ConstraintMatrices, ConstraintSynthesizer, ConstraintSystem, ConstraintSystemRef, Matrix, OptimizationGoal,
    Result as R1CSResult, SynthesisError,
};
use ark_std::{
    cell::RefCell,
    collections::BTreeMap,
    marker::PhantomData,
    rand::{Rng, RngCore},
    vec::Vec,
};
use core::ffi::CStr;

// ---------------------------------------------------------------------------------------------------------------------
// status codes -> SynthesisError (the library never unwinds across the ABI; the reference builds with panic = 'abort')
// ---------------------------------------------------------------------------------------------------------------------
fn status(rc: i32) -> R1CSResult<()> {
    match rc {
        sys::G16_OK => Ok(()),
        sys::G16_ERR_POLYNOMIAL_DEGREE_TOO_LARGE => Err(SynthesisError::PolynomialDegreeTooLarge), // r1cs_to_qap.rs:134,179
        sys::G16_ERR_MALFORMED_KEY => Err(SynthesisError::MalformedVerifyingKey),                  // verifier.rs:30
        _ => {
            // G16_ERR_BAD_ARGUMENT / G16_ERR_CUDA carry a message; SynthesisError has no string variant
            let msg = unsafe { CStr::from_ptr(sys::g16_last_error()) }.to_string_lossy().into_owned();
            eprintln!("libg16b200: {msg}");
            Err(SynthesisError::Unsatisfiable)
        },
    }
}

/// Curve id of the C ABI from the scalar-field modulus (the three curves the library is built for).
pub fn curve_id<F: PrimeField>() -> Option<i32> {
    let m = F::MODULUS.as_ref();
    match (F::MODULUS_BIT_SIZE, m[0]) {
        (255, 0xffff_ffff_0000_0001) => Some(sys::G16_CURVE_BLS12_381),
        (254, 0x43e1_f593_f000_0001) => Some(sys::G16_CURVE_BN254),
        (253, 0x0a11_8000_0000_0001) => Some(sys::G16_CURVE_BLS12_377),
        _ => None,
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// packing helpers
// ---------------------------------------------------------------------------------------------------------------------
/// Montgomery limbs of a prime-field element, exactly as ark-ff keeps them in memory.
/// SAFETY: every `Fp<MontBackend<_, N>, N>` is `BigInt<N>([u64; N])` followed by a zero-sized marker.
fn fp_limbs<F: PrimeField>(x: &F) -> &[u64] {
    debug_assert_eq!(core::mem::size_of::<F>() % 8, 0);
    unsafe { core::slice::from_raw_parts(x as *const F as *const u64, core::mem::size_of::<F>() / 8) }
}
fn fp_from_limbs<F: PrimeField>(l: &[u64]) -> F {
    let mut x = F::zero();
    debug_assert_eq!(core::mem::size_of::<F>(), 8 * l.len());
    unsafe { core::ptr::copy_nonoverlapping(l.as_ptr(), &mut x as *mut F as *mut u64, l.len()) };
    x
}
/// `&[F]` of scalars as the ABI wants them: no copy.
fn scalars_ptr<F: PrimeField>(xs: &[F]) -> *const u64 {
    xs.as_ptr() as *const u64
}
/// x || y of a short-Weierstrass affine point over Fq (one prime-field element per coordinate) or Fq2 (two), zeros for
/// the point at infinity.  `to_base_prime_field_elements` yields c0 then c1 for a quadratic extension.
fn push_point<P: SWCurveConfig>(out: &mut Vec<u64>, p: &Affine<P>, limbs_per_point: usize) {
    if p.infinity {
        out.extend(core::iter::repeat(0u64).take(limbs_per_point));
        return;
    }
    for coord in [&p.x, &p.y] {
        for c in coord.to_base_prime_field_elements() {
            out.extend_from_slice(fp_limbs(&c));
        }
    }
}
fn point_limbs<P: SWCurveConfig>() -> usize {
    let fq = core::mem::size_of::<<P::BaseField as Field>::BasePrimeField>() / 8;
    2 * fq * P::BaseField::extension_degree() as usize
}
pub fn pack_points<P: SWCurveConfig>(ps: &[Affine<P>]) -> Vec<u64> {
    let w = point_limbs::<P>();
    let mut out = Vec::with_capacity(ps.len() * w);
    for p in ps {
        push_point(&mut out, p, w);
    }
    out
}
pub fn unpack_point<P: SWCurveConfig>(l: &[u64]) -> Affine<P> {
    if l.iter().all(|&w| w == 0) {
        return Affine::<P>::identity();
    }
    let deg = P::BaseField::extension_degree() as usize;
    let fq = l.len() / (2 * deg);
    let coord = |k: usize| {
        let elems: Vec<<P::BaseField as Field>::BasePrimeField> =
            (0..deg).map(|i| fp_from_limbs(&l[(k * deg + i) * fq..(k * deg + i + 1) * fq])).collect();
        P::BaseField::from_base_prime_field_elems(elems).expect("coordinate")
    };
    Affine::<P>::new_unchecked(coord(0), coord(1))
}

/// `ConstraintMatrices` rows (`Vec<Vec<(F, usize)>>`) -> CSR arrays of the ABI (`g16_csr`).
pub struct Csr {
    row_ptr: Vec<u32>,
    col: Vec<u32>,
    val: Vec<u64>,
}
impl Csr {
    pub fn new<F: PrimeField>(m: &Matrix<F>) -> Self {
        let nnz: usize = m.iter().map(|r| r.len()).sum();
        let mut s = Csr { row_ptr: Vec::with_capacity(m.len() + 1), col: Vec::with_capacity(nnz), val: Vec::with_capacity(4 * nnz) };
        s.row_ptr.push(0);
        for row in m {
            for (coeff, idx) in row {
                s.col.push(*idx as u32);
                s.val.extend_from_slice(fp_limbs(coeff));
            }
            s.row_ptr.push(s.col.len() as u32);
        }
        s
    }
    fn desc(&self) -> sys::g16_csr {
        sys::g16_csr { row_ptr: self.row_ptr.as_ptr(), col: self.col.as_ptr(), val: self.val.as_ptr() }
    }
}

/// The pairing engines whose groups are short-Weierstrass curves (all of ark-bls12-381 / ark-bn254 / ark-bls12-377).
pub trait SwPairing: Pairing<G1Affine = Affine<Self::G1Config>, G2Affine = Affine<Self::G2Config>> {
    type G1Config: SWCurveConfig;
    type G2Config: SWCurveConfig;
}
impl<E, P1, P2> SwPairing for E
where
    P1: SWCurveConfig,
    P2: SWCurveConfig,
    E: Pairing<G1Affine = Affine<P1>, G2Affine = Affine<P2>>,
{
    type G1Config = P1;
    type G2Config = P2;
}

// ---------------------------------------------------------------------------------------------------------------------
// the prover: one context = one curve on one GPU with ONE circuit and ONE proving key resident
// ---------------------------------------------------------------------------------------------------------------------
pub struct B200Prover<E: SwPairing> {
    ctx: *mut sys::g16_ctx,
    num_inputs: usize,
    num_constraints: usize,
    num_variables: usize,
    fq_limbs: usize,
    _e: PhantomData<E>,
}
// the context is used by one thread at a time (include/g16b200.h); moving it between threads is fine
unsafe impl<E: SwPairing> Send for B200Prover<E> {}

impl<E: SwPairing> Drop for B200Prover<E> {
    fn drop(&mut self) {
        unsafe { sys::g16_ctx_destroy(self.ctx) }
    }
}

impl<E: SwPairing> B200Prover<E> {
    /// Once per circuit: `ConstraintMatrices` -> CSR, `ProvingKey` -> packed queries; both stay resident on the GPU.
    /// `rank` / `world`: this process's share of a multi-GPU proof (pair i of every MSM lives on rank i mod world).
    pub fn new(device: i32, matrices: &ConstraintMatrices<E::ScalarField>, pk: &ProvingKey<E>, rank: u32, world: u32) -> R1CSResult<Self> {
        let curve = curve_id::<E::ScalarField>().ok_or(SynthesisError::Unsatisfiable)?;
        let mut ctx = core::ptr::null_mut();
        status(unsafe { sys::g16_ctx_create(curve, device, &mut ctx) })?;
        let me = Self {
            ctx,
            num_inputs: matrices.num_instance_variables,
            num_constraints: matrices.num_constraints,
            num_variables: matrices.num_instance_variables + matrices.num_witness_variables,
            fq_limbs: unsafe { sys::g16_fq_limbs(ctx) } as usize,
            _e: PhantomData,
        };
        let (a, b, c) = (Csr::new(&matrices.a), Csr::new(&matrices.b), Csr::new(&matrices.c));
        status(unsafe {
            sys::g16_circuit_load(
                ctx,
                matrices.num_instance_variables as u32,
                matrices.num_constraints as u32,
                matrices.num_witness_variables as u32,
                &a.desc(),
                &b.desc(),
                &c.desc(),
            )
        })?;
        me.load_proving_key(pk, rank, world)?;
        Ok(me)
    }

    /// data_structures.rs:126-143 -> g16_pk_load.  The queries are the FULL ark vectors (a_query[0] included).
    pub fn load_proving_key(&self, pk: &ProvingKey<E>, rank: u32, world: u32) -> R1CSResult<()> {
        let aq = pack_points(&pk.a_query);
        let b1 = pack_points(&pk.b_g1_query);
        let b2 = pack_points(&pk.b_g2_query);
        let hq = pack_points(&pk.h_query);
        let lq = pack_points(&pk.l_query);
        let alpha_g1 = pack_points(&[pk.vk.alpha_g1]);
        let beta_g1 = pack_points(&[pk.beta_g1]);
        let delta_g1 = pack_points(&[pk.delta_g1]);
        let beta_g2 = pack_points(&[pk.vk.beta_g2]);
        let delta_g2 = pack_points(&[pk.vk.delta_g2]);
        let desc = sys::g16_pk_desc {
            a_query: aq.as_ptr(),
            a_len: pk.a_query.len() as u64,
            b_g1_query: b1.as_ptr(),
            b_g1_len: pk.b_g1_query.len() as u64,
            b_g2_query: b2.as_ptr(),
            b_g2_len: pk.b_g2_query.len() as u64,
            h_query: hq.as_ptr(),
            h_len: pk.h_query.len() as u64,
            l_query: lq.as_ptr(),
            l_len: pk.l_query.len() as u64,
            alpha_g1: alpha_g1.as_ptr(),
            beta_g1: beta_g1.as_ptr(),
            delta_g1: delta_g1.as_ptr(),
            beta_g2: beta_g2.as_ptr(),
            delta_g2: delta_g2.as_ptr(),
        };
        status(unsafe { sys::g16_pk_load(self.ctx, &desc, rank, world) })
    }

    fn proof_from_limbs(&self, out: &[u64]) -> Proof<E> {
        let n = self.fq_limbs;
        Proof { a: unpack_point(&out[..2 * n]), b: unpack_point(&out[2 * n..6 * n]), c: unpack_point(&out[6 * n..8 * n]) }
    }

    /// Drop-in for `Groth16::<E>::create_proof_with_reduction_and_matrices` (src/prover.rs:26-51).  `pk` and `matrices` are
    /// the ones made resident by `new`; they are accepted (and their sizes checked) so that call sites read the same.
    #[allow(clippy::too_many_arguments)]
    pub fn create_proof_with_reduction_and_matrices(
        &self,
        _pk: &ProvingKey<E>,
        r: E::ScalarField,
        s: E::ScalarField,
        _matrices: &ConstraintMatrices<E::ScalarField>,
        num_inputs: usize,
        num_constraints: usize,
        full_assignment: &[E::ScalarField],
    ) -> R1CSResult<Proof<E>> {
        if num_inputs != self.num_inputs || num_constraints != self.num_constraints || full_assignment.len() != self.num_variables {
            return Err(SynthesisError::MalformedVerifyingKey);
        }
        let mut out = ark_std::vec![0u64; 8 * self.fq_limbs];
        status(unsafe {
            sys::g16_prove(self.ctx, fp_limbs(&r).as_ptr(), fp_limbs(&s).as_ptr(), scalars_ptr(full_assignment), 0, out.as_mut_ptr())
        })?;
        Ok(self.proof_from_limbs(&out))
    }

    /// src/prover.rs:173-204: synthesize, then prove with the given randomness.
    pub fn create_proof_with_reduction<C: ConstraintSynthesizer<E::ScalarField>>(
        &self,
        circuit: C,
        pk: &ProvingKey<E>,
        r: E::ScalarField,
        s: E::ScalarField,
    ) -> R1CSResult<Proof<E>> {
        let cs = ConstraintSystem::new_ref();
        cs.set_optimization_goal(OptimizationGoal::Constraints);
        circuit.generate_constraints(cs.clone())?;
        debug_assert!(cs.is_satisfied().unwrap());
        cs.finalize();
        let matrices = cs.to_matrices().ok_or(SynthesisError::AssignmentMissing)?;
        let prover = cs.borrow().ok_or(SynthesisError::AssignmentMissing)?;
        let full_assignment = [prover.instance_assignment.as_slice(), prover.witness_assignment.as_slice()].concat();
        self.create_proof_with_reduction_and_matrices(
            pk,
            r,
            s,
            &matrices,
            prover.instance_assignment.len(),
            cs.num_constraints(),
            &full_assignment,
        )
    }
    /// src/prover.rs:155-170
    pub fn create_proof_with_reduction_no_zk<C: ConstraintSynthesizer<E::ScalarField>>(&self, circuit: C, pk: &ProvingKey<E>) -> R1CSResult<Proof<E>> {
        self.create_proof_with_reduction(circuit, pk, E::ScalarField::zero(), E::ScalarField::zero())
    }
    /// src/prover.rs:138-152: `r` is sampled before `s` (matters when an RNG is replayed, prover.rs:146-147).
    pub fn create_random_proof_with_reduction<C: ConstraintSynthesizer<E::ScalarField>>(
        &self,
        circuit: C,
        pk: &ProvingKey<E>,
        rng: &mut impl Rng,
    ) -> R1CSResult<Proof<E>> {
        let r = E::ScalarField::rand(rng);
        let s = E::ScalarField::rand(rng);
        self.create_proof_with_reduction(circuit, pk, r, s)
    }

    /// Multi-GPU, first half: this rank's five partial MSM sums ([h, l, a, b_g1] G1 affine, then b_g2 G2 affine).
    pub fn prove_partial(&self, r: E::ScalarField, full_assignment: &[E::ScalarField]) -> R1CSResult<Vec<u64>> {
        let mut out = ark_std::vec![0u64; unsafe { sys::g16_partial_limbs(self.ctx) } as usize];
        status(unsafe { sys::g16_prove_partial(self.ctx, fp_limbs(&r).as_ptr(), scalars_ptr(full_assignment), 0, out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Multi-GPU, second half: all ranks' partial records (rank order), gathered by the caller (MPI / NCCL all-gather).
    pub fn prove_assemble(&self, r: E::ScalarField, s: E::ScalarField, partials: &[u64], nparts: u32) -> R1CSResult<Proof<E>> {
        let mut out = ark_std::vec![0u64; 8 * self.fq_limbs];
        status(unsafe {
            sys::g16_prove_assemble(self.ctx, fp_limbs(&r).as_ptr(), fp_limbs(&s).as_ptr(), partials.as_ptr(), nparts, out.as_mut_ptr())
        })?;
        Ok(self.proof_from_limbs(&out))
    }

    /// `VariableBaseMSM::msm_bigint` on G1 (call sites src/prover.rs:66,74,262): truncates to the shorter operand like ark.
    pub fn msm_g1(&self, bases: &[E::G1Affine], scalars: &[<E::ScalarField as PrimeField>::BigInt]) -> R1CSResult<E::G1> {
        let n = bases.len().min(scalars.len());
        let b = pack_points(&bases[..n]);
        let mut out = ark_std::vec![0u64; 3 * self.fq_limbs];
        status(unsafe { sys::g16_msm_g1(self.ctx, b.as_ptr(), scalars.as_ptr() as *const u64, n as u64, out.as_mut_ptr()) })?;
        // X || Y || Z normalised to Z = 1 (identity: Z = 0)
        let nl = self.fq_limbs;
        if out[2 * nl..].iter().all(|&w| w == 0) {
            return Ok(E::G1::zero());
        }
        Ok(unpack_point::<E::G1Config>(&out[..2 * nl]).into())
    }

    pub fn timings(&self) -> sys::g16_timings {
        let mut t = sys::g16_timings::default();
        unsafe { sys::g16_get_timings(self.ctx, &mut t) };
        t
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// NTT path only: an R1CSToQAP that ark-groth16 accepts as its second type parameter (src/lib.rs:55)
// ---------------------------------------------------------------------------------------------------------------------
pub struct GpuReduction;

struct ThreadCtx {
    ctx: *mut sys::g16_ctx,
    loaded: Option<(usize, usize, usize, usize)>, // (instance vars, witness vars, constraints, nnz(a)) of the resident circuit
}
thread_local! {
    static CTXS: RefCell<BTreeMap<i32, ThreadCtx>> = RefCell::new(BTreeMap::new());
}
/// One context per (curve, thread), created on first use on device `G16B200_DEVICE` (default 0) and kept.
fn with_thread_ctx<F: PrimeField, T>(f: impl FnOnce(&mut ThreadCtx) -> R1CSResult<T>) -> R1CSResult<T> {
    let curve = curve_id::<F>().ok_or(SynthesisError::Unsatisfiable)?;
    CTXS.with(|m| {
        let mut m = m.borrow_mut();
        if !m.contains_key(&curve) {
            let device = std::env::var("G16B200_DEVICE").ok().and_then(|v| v.parse().ok()).unwrap_or(0);
            let mut ctx = core::ptr::null_mut();
            status(unsafe { sys::g16_ctx_create(curve, device, &mut ctx) })?;
            m.insert(curve, ThreadCtx { ctx, loaded: None });
        }
        f(m.get_mut(&curve).unwrap())
    })
}
fn load_matrices_once<F: PrimeField>(t: &mut ThreadCtx, m: &ConstraintMatrices<F>) -> R1CSResult<()> {
    let key = (m.num_instance_variables, m.num_witness_variables, m.num_constraints, m.a_num_non_zero);
    if t.loaded == Some(key) {
        return Ok(());
    }
    let (a, b, c) = (Csr::new(&m.a), Csr::new(&m.b), Csr::new(&m.c));
    status(unsafe {
        sys::g16_circuit_load(
            t.ctx,
            m.num_instance_variables as u32,
            m.num_constraints as u32,
            m.num_witness_variables as u32,
            &a.desc(),
            &b.desc(),
            &c.desc(),
        )
    })?;
    t.loaded = Some(key);
    Ok(())
}

impl R1CSToQAP for GpuReduction {
    fn instance_map_with_evaluation<F: PrimeField, D: EvaluationDomain<F>>(
        cs: ConstraintSystemRef<F>,
        t: &F,
    ) -> Result<(Vec<F>, Vec<F>, Vec<F>, F, usize, usize), SynthesisError> {
        LibsnarkReduction::instance_map_with_evaluation::<F, D>(cs, t) // setup side: unchanged (src/r1cs_to_qap.rs:128-170)
    }

    fn witness_map_from_matrices<F: PrimeField, D: EvaluationDomain<F>>(
        matrices: &ConstraintMatrices<F>,
        num_inputs: usize,
        num_constraints: usize,
        full_assignment: &[F],
    ) -> R1CSResult<Vec<F>> {
        with_thread_ctx::<F, _>(|t| {
            load_matrices_once(t, matrices)?;
            let n = (num_constraints + num_inputs).next_power_of_two();
            let mut h = ark_std::vec![F::zero(); n];
            status(unsafe { sys::g16_witness_map(t.ctx, scalars_ptr(full_assignment), 0, h.as_mut_ptr() as *mut u64) })?;
            Ok(h)
        })
    }

    fn h_query_scalars<F: PrimeField, D: EvaluationDomain<F>>(
        max_power: usize,
        t: F,
        zt: F,
        delta_inverse: F,
    ) -> Result<Vec<F>, SynthesisError> {
        LibsnarkReduction::h_query_scalars::<F, D>(max_power, t, zt, delta_inverse) // src/r1cs_to_qap.rs:237-247
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// impl SNARK, mirroring src/lib.rs:59-97: setup and verification forward to ark-groth16, proving goes to the GPU
// ---------------------------------------------------------------------------------------------------------------------
pub struct Groth16B200<E: SwPairing> {
    _p: PhantomData<E>,
}

impl<E: SwPairing> SNARK<E::ScalarField> for Groth16B200<E> {
    type ProvingKey = ProvingKey<E>;
    type VerifyingKey = VerifyingKey<E>;
    type Proof = Proof<E>;
    type ProcessedVerifyingKey = PreparedVerifyingKey<E>;
    type Error = SynthesisError;

    fn circuit_specific_setup<C: ConstraintSynthesizer<E::ScalarField>, R: RngCore>(
        circuit: C,
        rng: &mut R,
    ) -> Result<(Self::ProvingKey, Self::VerifyingKey), Self::Error> {
        Groth16::<E>::circuit_specific_setup(circuit, rng)
    }

    /// One-shot form (uploads the circuit and the key for this single proof): fine for tests, wasteful in production --
    /// keep a [`B200Prover`] alive per circuit instead.
    fn prove<C: ConstraintSynthesizer<E::ScalarField>, R: RngCore>(
        pk: &Self::ProvingKey,
        circuit: C,
        rng: &mut R,
    ) -> Result<Self::Proof, Self::Error> {
        let cs = ConstraintSystem::new_ref();
        cs.set_optimization_goal(OptimizationGoal::Constraints);
        circuit.generate_constraints(cs.clone())?;
        cs.finalize();
        let matrices = cs.to_matrices().ok_or(SynthesisError::AssignmentMissing)?;
        let device = std::env::var("G16B200_DEVICE").ok().and_then(|v| v.parse().ok()).unwrap_or(0);
        let prover = B200Prover::<E>::new(device, &matrices, pk, 0, 1)?;
        let r = E::ScalarField::rand(rng);
        let s = E::ScalarField::rand(rng);
        let asg = cs.borrow().ok_or(SynthesisError::AssignmentMissing)?;
        let full_assignment = [asg.instance_assignment.as_slice(), asg.witness_assignment.as_slice()].concat();
        prover.create_proof_with_reduction_and_matrices(pk, r, s, &matrices, asg.instance_assignment.len(), cs.num_constraints(), &full_assignment)
    }

    fn process_vk(circuit_vk: &Self::VerifyingKey) -> Result<Self::ProcessedVerifyingKey, Self::Error> {
        Groth16::<E>::process_vk(circuit_vk)
    }

    fn verify_with_processed_vk(
        circuit_pvk: &Self::ProcessedVerifyingKey,
        x: &[E::ScalarField],
        proof: &Self::Proof,
    ) -> Result<bool, Self::Error> {
        Groth16::<E>::verify_with_processed_vk(circuit_pvk, x, proof)
    }
}

impl<E: SwPairing> CircuitSpecificSetupSNARK<E::ScalarField> for Groth16B200<E> {}

#[cfg(test)]
mod tests {
    //! The reference's own round trip (src/test.rs:45-72) with the GPU prover and ark's verifier, plus bit-equality with
    //! ark's CPU prover for fixed (r, s).  Needs an H100 and libg16b200.so at run time.
    use super::*;
    use ark_bls12_381::{Bls12_381, Fr};
    use ark_relations::{lc, r1cs::Variable};
    use ark_std::test_rng;

    struct MySillyCircuit {
        a: Option<Fr>,
        b: Option<Fr>,
    }
    impl ConstraintSynthesizer<Fr> for MySillyCircuit {
        fn generate_constraints(self, cs: ConstraintSystemRef<Fr>) -> Result<(), SynthesisError> {
            let a = cs.new_witness_variable(|| self.a.ok_or(SynthesisError::AssignmentMissing))?;
            let b = cs.new_witness_variable(|| self.b.ok_or(SynthesisError::AssignmentMissing))?;
            let c = cs.new_input_variable(|| Ok(self.a.unwrap() * self.b.unwrap()))?;
            for _ in 0..6 {
                cs.enforce_constraint(lc!() + a, lc!() + b, lc!() + c)?;
            }
            let _ = Variable::One;
            Ok(())
        }
    }

    #[test]
    fn gpu_proof_equals_cpu_proof_and_verifies() {
        let rng = &mut test_rng();
        let (pk, vk) = Groth16::<Bls12_381>::circuit_specific_setup(MySillyCircuit { a: None, b: None }, rng).unwrap();
        let (a, b) = (Fr::rand(rng), Fr::rand(rng));
        let (r, s) = (Fr::rand(rng), Fr::rand(rng));
        let cpu = Groth16::<Bls12_381>::create_proof_with_reduction(MySillyCircuit { a: Some(a), b: Some(b) }, &pk, r, s).unwrap();
        let cs = ConstraintSystem::new_ref();
        MySillyCircuit { a: Some(a), b: Some(b) }.generate_constraints(cs.clone()).unwrap();
        cs.finalize();
        let prover = B200Prover::<Bls12_381>::new(0, &cs.to_matrices().unwrap(), &pk, 0, 1).unwrap();
        let gpu = prover.create_proof_with_reduction(MySillyCircuit { a: Some(a), b: Some(b) }, &pk, r, s).unwrap();
        assert_eq!(cpu, gpu);
        assert!(Groth16::<Bls12_381>::verify(&vk, &[a * b], &gpu).unwrap());
    }
}
