//! `ark-groth16-b200`: ark-groth16 0.5's prover API on top of `libg16b200.so` (H100 / sm_90a CUDA kernels).
//!
//! What is replaced (file:line of arkworks-rs/groth16 @ d570ee5):
//!   * `Groth16::<E>::create_proof_with_reduction_and_matrices`   src/prover.rs:26-51   -> [`B200Prover::create_proof_with_reduction_and_matrices`]
//!   * `Groth16::<E>::create_proof_with_reduction` / `_no_zk` / `create_random_proof_with_reduction`
//!                                                                  src/prover.rs:138-204 -> methods of the same names
//!   * `impl SNARK for Groth16<E, QAP>`                             src/lib.rs:59-97      -> [`Groth16B200`] (setup / verify forwarded)
//!   * `R1CSToQAP::witness_map_from_matrices`                       src/r1cs_to_qap.rs:172-235 -> [`GpuReduction`] (NTT path only,
//!     selectable as `ark_groth16::Groth16<E, GpuReduction>` without touching the MSMs)
//!   * ark-circom's `CircomReduction` (circom circuits, snarkjs-compatible keys)  -> [`GpuCircomReduction`] for
//!     `ark_groth16::Groth16<E, GpuCircomReduction>` (setup and witness map), and [`B200Prover::new_with_qap`] with
//!     `sys::G16_QAP_CIRCOM` for the whole proof
//!   * ark-circom's `read_zkey` (snarkjs `.zkey` files) followed by `Groth16<E, CircomReduction>` -> [`B200Prover::load_zkey`]
//!   * ark-circom's `R1CSFile` + `CircomCircuit` (circom `.r1cs` files, all three matrices) -> [`B200Prover::load_r1cs`], the
//!     key of a `.zkey` onto it -> [`B200Prover::load_zkey_key`], and `read_witness` (`.wtns`) -> [`B200Prover::read_wtns`]
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
use ark_serialize::{Compress, SerializationError, Validate};
use ark_relations::r1cs::{
    ConstraintMatrices, ConstraintSynthesizer, ConstraintSystem, ConstraintSystemRef, Matrix, OptimizationGoal,
    Result as R1CSResult, SynthesisError,
};
use ark_std::{
    cell::{Cell, RefCell},
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
        sys::G16_ERR_UNSATISFIED => {
            // G16_CHECK_WITNESS refused the assignment; the message names the constraint or element
            let msg = unsafe { CStr::from_ptr(sys::g16_last_error()) }.to_string_lossy().into_owned();
            eprintln!("libg16b200: {msg}");
            Err(SynthesisError::Unsatisfiable)
        },
        _ => {
            // G16_ERR_BAD_ARGUMENT / G16_ERR_CUDA carry a message; SynthesisError has no string variant
            let msg = unsafe { CStr::from_ptr(sys::g16_last_error()) }.to_string_lossy().into_owned();
            eprintln!("libg16b200: {msg}");
            Err(SynthesisError::Unsatisfiable)
        },
    }
}

/// status codes of the serialized-key calls -> SerializationError.  A rejected key (G16_ERR_INVALID_DATA, and a
/// gamma_abc_g1 / query length that does not fit the circuit, G16_ERR_MALFORMED_KEY) is `InvalidData`, whose message naming
/// the member, index and reason goes to stderr; a CUDA failure or a bad argument is an `IoError` carrying the library's
/// message, so that callers can tell a missing GPU from bad key data.
/// nPublic + 1 from section 2 of a `.zkey` (n8q-byte base field), found by walking the section table; 1 when the file is
/// too broken to say (g16_zkey_load then refuses it before writing anything).
fn zkey_num_inputs(b: &[u8], n8q: usize) -> usize {
    let u32_at = |o: usize| -> Option<usize> { b.get(o..o + 4).map(|s| u32::from_le_bytes([s[0], s[1], s[2], s[3]]) as usize) };
    let u64_at = |o: usize| -> Option<usize> {
        b.get(o..o + 8).map(|s| u64::from_le_bytes([s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7]]) as usize)
    };
    let mut pos = 12usize;
    for _ in 0..u32_at(8).unwrap_or(0) {
        let (Some(id), Some(size)) = (u32_at(pos), u64_at(pos + 4)) else { return 1 };
        pos += 12;
        if id == 2 {
            if u32_at(pos) != Some(n8q) {
                return 1;
            }
            let Some(n8r) = u32_at(pos + 4 + n8q) else { return 1 };
            return u32_at(pos + 8 + n8q + n8r + 4).map_or(1, |p| p + 1);
        }
        pos = pos.saturating_add(size);
    }
    1
}

fn ser_status(rc: i32) -> Result<(), SerializationError> {
    if rc == sys::G16_OK {
        return Ok(());
    }
    let msg = unsafe { CStr::from_ptr(sys::g16_last_error()) }.to_string_lossy().into_owned();
    match rc {
        sys::G16_ERR_INVALID_DATA | sys::G16_ERR_MALFORMED_KEY => {
            eprintln!("libg16b200: {msg}");
            Err(SerializationError::InvalidData)
        },
        _ => Err(SerializationError::IoError(ark_std::io::Error::new(ark_std::io::ErrorKind::Other, msg))),
    }
}

/// Curve id of the C ABI from the scalar-field modulus (the four curves the library is built for).
pub fn curve_id<F: PrimeField>() -> Option<i32> {
    let m = F::MODULUS.as_ref();
    match (F::MODULUS_BIT_SIZE, m[0]) {
        (255, 0xffff_ffff_0000_0001) => Some(sys::G16_CURVE_BLS12_381),
        (254, 0x43e1_f593_f000_0001) => Some(sys::G16_CURVE_BN254),
        (253, 0x0a11_8000_0000_0001) => Some(sys::G16_CURVE_BLS12_377),
        (377, 0x8508_c000_0000_0001) => Some(sys::G16_CURVE_BW6_761),
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
        let mut s = Csr { row_ptr: Vec::with_capacity(m.len() + 1), col: Vec::with_capacity(nnz), val: Vec::with_capacity(core::mem::size_of::<F>() / 8 * nnz) };
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

/// A powers-of-tau transcript (phase 1 of a Groth16 ceremony): tau_g1[i] = [tau^i]G1, tau_g2[i] = [tau^i]G2,
/// alpha_tau_g1[i] = [alpha tau^i]G1, beta_tau_g1[i] = [beta tau^i]G1, beta_g2 = [beta]G2.
pub struct PowersOfTau<E: SwPairing> {
    pub tau_g1: Vec<Affine<E::G1Config>>,
    pub tau_g2: Vec<Affine<E::G2Config>>,
    pub alpha_tau_g1: Vec<Affine<E::G1Config>>,
    pub beta_tau_g1: Vec<Affine<E::G1Config>>,
    pub beta_g2: Affine<E::G2Config>,
}

/// What `B200Prover::read_ptau` read from a snarkjs `.ptau` file: its header, the transcript, and for a prepared file read
/// for a domain one level of Lagrange points.
pub struct Ptau<E: SwPairing> {
    pub power: u32,
    pub ceremony_power: u32,
    pub prepared: bool,
    pub srs: PowersOfTau<E>,
    pub lagrange: Option<LagrangePoints<E>>,
}

/// Level `log_n` of a prepared `.ptau` file's Lagrange points: tau_g1[i] = [L_i(tau)]G1, tau_g2[i] = [L_i(tau)]G2,
/// alpha_tau_g1[i] = [alpha L_i(tau)]G1, beta_tau_g1[i] = [beta L_i(tau)]G1 over the domain of 2^log_n points, and
/// tau_g1_h the odd entries of level log_n + 1: the CircomReduction H query at delta = 1 when that level is the file's top
/// one, and with `h_over_2n` (an interior level, over 2n powers) that query plus (omega_2n^(2i+1) / 2n) [tau^(2n-1)].
pub struct LagrangePoints<E: SwPairing> {
    pub log_n: u32,
    pub h_over_2n: bool,
    pub tau_g1: Vec<Affine<E::G1Config>>,
    pub tau_g2: Vec<Affine<E::G2Config>>,
    pub alpha_tau_g1: Vec<Affine<E::G1Config>>,
    pub beta_tau_g1: Vec<Affine<E::G1Config>>,
    pub tau_g1_h: Vec<Affine<E::G1Config>>,
}

/// One contribution's public record (the public key of Bowe, Gabizon and Miers, as snarkjs and bellman's phase2 publish it):
/// `after_g1` = x D for the running point D (phase 2: delta_g1; phase 1: tau_g1[1], alpha_tau_g1[0], beta_tau_g1[0]),
/// `s_x_g1` = x s for a G1 point `s` of the contributor's choice, `r_x_g2` = x r.  `r_g2` must be the checker's own hash to
/// G2 of the contribution's transcript, never a point taken from the contributor: an r with a known discrete log makes the
/// proof of knowledge empty.  The hash and the file format that binds it are the caller's.
pub struct ContributionRecord<E: SwPairing> {
    pub after_g1: Affine<E::G1Config>,
    pub s_g1: Affine<E::G1Config>,
    pub s_x_g1: Affine<E::G1Config>,
    pub r_g2: Affine<E::G2Config>,
    pub r_x_g2: Affine<E::G2Config>,
}
impl<E: SwPairing> ContributionRecord<E> {
    /// The contributor's record for secret `x`: `after` is its new running point, `s` its chosen point, `r` the hash to G2
    /// of its contribution's transcript; s_x_g1 = x s and r_x_g2 = x r are formed here.
    pub fn make(x: E::ScalarField, after: Affine<E::G1Config>, s: Affine<E::G1Config>, r: Affine<E::G2Config>) -> Self {
        let k = x.into_bigint();
        ContributionRecord {
            after_g1: after,
            s_g1: s,
            s_x_g1: Affine::<E::G1Config>::from(s.mul_bigint(k)),
            r_g2: r,
            r_x_g2: Affine::<E::G2Config>::from(r.mul_bigint(k)),
        }
    }
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
    g2_limbs: usize,   // one G2 affine point: 4 * fq_limbs over Fq2, 2 * fq_limbs on BW6-761 (G2 over Fq)
    flags: Cell<u32>,  // ored into every prove call: G16_CHECK_WITNESS after set_check_witness(true)
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
    /// The circuit is proved under `LibsnarkReduction`, ark-groth16's default (`new_with_qap` names another).
    pub fn new(device: i32, matrices: &ConstraintMatrices<E::ScalarField>, pk: &ProvingKey<E>, rank: u32, world: u32) -> R1CSResult<Self> {
        Self::new_with_qap(device, sys::G16_QAP_LIBSNARK, matrices, pk, rank, world)
    }

    /// `new` under the R1CS-to-QAP reduction `qap` (`sys::G16_QAP_LIBSNARK` or `sys::G16_QAP_CIRCOM`), the counterpart of
    /// the second type parameter of `Groth16<E, QAP>`: a key made by `Groth16<E, CircomReduction>` (or
    /// `Groth16<E, GpuCircomReduction>`) is proved with `sys::G16_QAP_CIRCOM`.
    pub fn new_with_qap(
        device: i32,
        qap: i32,
        matrices: &ConstraintMatrices<E::ScalarField>,
        pk: &ProvingKey<E>,
        rank: u32,
        world: u32,
    ) -> R1CSResult<Self> {
        let curve = curve_id::<E::ScalarField>().ok_or(SynthesisError::Unsatisfiable)?;
        let mut ctx = core::ptr::null_mut();
        status(unsafe { sys::g16_ctx_create(curve, device, &mut ctx) })?;
        let me = Self {
            ctx,
            num_inputs: matrices.num_instance_variables,
            num_constraints: matrices.num_constraints,
            num_variables: matrices.num_instance_variables + matrices.num_witness_variables,
            fq_limbs: unsafe { sys::g16_fq_limbs(ctx) } as usize,
            g2_limbs: unsafe { sys::g16_g2_limbs(ctx) } as usize,
            flags: Cell::new(0),
            _e: PhantomData,
        };
        let (a, b, c) = (Csr::new(&matrices.a), Csr::new(&matrices.b), Csr::new(&matrices.c));
        status(unsafe {
            sys::g16_circuit_load_qap(
                ctx,
                qap,
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

    /// `ProvingKey::<E>::deserialize_with_mode(bytes, compress, validate)` and `new` in one step, decoded and validated on the
    /// GPU (g16_pk_load_serialized): `bytes` is a whole ark-serialized ProvingKey<E>.  Returns the prover and the key's
    /// VerifyingKey (whose bytes are the prefix of `bytes`).  Every rank decodes and validates all points.
    #[allow(clippy::too_many_arguments)]
    pub fn new_from_bytes(
        device: i32,
        qap: i32,
        matrices: &ConstraintMatrices<E::ScalarField>,
        bytes: &[u8],
        compress: Compress,
        validate: Validate,
        rank: u32,
        world: u32,
    ) -> Result<(Self, VerifyingKey<E>), SerializationError> {
        let curve = curve_id::<E::ScalarField>().ok_or_else(|| {
            SerializationError::IoError(ark_std::io::Error::new(ark_std::io::ErrorKind::Other, "libg16b200 does not support this curve"))
        })?;
        let mut ctx = core::ptr::null_mut();
        ser_status(unsafe { sys::g16_ctx_create(curve, device, &mut ctx) })?;
        let me = Self {
            ctx,
            num_inputs: matrices.num_instance_variables,
            num_constraints: matrices.num_constraints,
            num_variables: matrices.num_instance_variables + matrices.num_witness_variables,
            fq_limbs: unsafe { sys::g16_fq_limbs(ctx) } as usize,
            g2_limbs: unsafe { sys::g16_g2_limbs(ctx) } as usize,
            flags: Cell::new(0),
            _e: PhantomData,
        };
        let (a, b, c) = (Csr::new(&matrices.a), Csr::new(&matrices.b), Csr::new(&matrices.c));
        ser_status(unsafe {
            sys::g16_circuit_load_qap(
                ctx,
                qap,
                matrices.num_instance_variables as u32,
                matrices.num_constraints as u32,
                matrices.num_witness_variables as u32,
                &a.desc(),
                &b.desc(),
                &c.desc(),
            )
        })?;
        let vk = me.load_proving_key_bytes(bytes, compress, validate, rank, world)?;
        Ok((me, vk))
    }

    /// A prover for the circuit and proving key of a snarkjs Groth16 `.zkey` (circuit_final.zkey), both decoded and made
    /// resident on the GPU in one call (g16_zkey_load): the GPU counterpart of ark-circom's `read_zkey` followed by
    /// `Groth16<E, CircomReduction>`.  The circuit's A and B are built on the device (a `.zkey` has no C: the calls that
    /// need it refuse), its sizes are derived from the file, and proofs run under `sys::G16_QAP_CIRCOM`.  Returns the
    /// prover and the key's VerifyingKey.  BN254 and BLS12-381 only, the curves snarkjs writes; a malformed file is
    /// `SerializationError::InvalidData` with the library's message.
    pub fn load_zkey(device: i32, bytes: &[u8], validate: Validate, rank: u32, world: u32) -> Result<(Self, VerifyingKey<E>), SerializationError> {
        let curve = curve_id::<E::ScalarField>().ok_or_else(|| {
            SerializationError::IoError(ark_std::io::Error::new(ark_std::io::ErrorKind::Other, "libg16b200 does not support this curve"))
        })?;
        let mut ctx = core::ptr::null_mut();
        ser_status(unsafe { sys::g16_ctx_create(curve, device, &mut ctx) })?;
        let (fq_limbs, g2_limbs) = (unsafe { sys::g16_fq_limbs(ctx) } as usize, unsafe { sys::g16_g2_limbs(ctx) } as usize);
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let (mut alpha_g1, mut beta_g1, mut delta_g1) = (ark_std::vec![0u64; w1], ark_std::vec![0u64; w1], ark_std::vec![0u64; w1]);
        let (mut beta_g2, mut gamma_g2, mut delta_g2) = (ark_std::vec![0u64; w2], ark_std::vec![0u64; w2], ark_std::vec![0u64; w2]);
        let mut abc = ark_std::vec![0u64; w1 * zkey_num_inputs(bytes, 8 * fq_limbs)];
        let null = core::ptr::null_mut();
        let desc = sys::g16_pk_export_desc {
            a_query: null,
            b_g1_query: null,
            b_g2_query: null,
            h_query: null,
            l_query: null,
            alpha_g1: alpha_g1.as_mut_ptr(),
            beta_g1: beta_g1.as_mut_ptr(),
            delta_g1: delta_g1.as_mut_ptr(),
            beta_g2: beta_g2.as_mut_ptr(),
            gamma_g2: gamma_g2.as_mut_ptr(),
            delta_g2: delta_g2.as_mut_ptr(),
            gamma_abc_g1: abc.as_mut_ptr(),
        };
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        let mut info = sys::g16_zkey_info::default();
        let rc = unsafe { sys::g16_zkey_load(ctx, bytes.as_ptr(), bytes.len() as u64, flags, rank, world, &desc, &mut info) };
        if rc != 0 {
            let err = ser_status(rc);
            unsafe { sys::g16_ctx_destroy(ctx) };
            err?;
        }
        let me = Self {
            ctx,
            num_inputs: info.num_inputs as usize,
            num_constraints: info.num_constraints as usize,
            num_variables: (info.num_inputs + info.num_witness) as usize,
            fq_limbs,
            g2_limbs,
            flags: Cell::new(0),
            _e: PhantomData,
        };
        let vk = VerifyingKey {
            alpha_g1: unpack_point(&alpha_g1),
            beta_g2: unpack_point(&beta_g2),
            gamma_g2: unpack_point(&gamma_g2),
            delta_g2: unpack_point(&delta_g2),
            gamma_abc_g1: abc.chunks(w1).take(info.num_inputs as usize).map(|l| unpack_point(l)).collect(),
        };
        Ok((me, vk))
    }

    /// A prover for the circuit of a circom `.r1cs` (circuit.r1cs), read on the GPU with all three matrices
    /// (g16_r1cs_load): the counterpart of ark-circom's `R1CSFile` followed by `CircomCircuit`, under the reduction `qap`.
    /// No key is resident yet: follow with `load_zkey_key`, `load_proving_key` or `setup_from_srs`.  Every call that reads
    /// C (`check_witness`, `set_check_witness`, `setup_from_srs`, `key_verification_pairs`) works on it.  A malformed file
    /// is `SerializationError::InvalidData` with the library's message.
    pub fn load_r1cs(device: i32, bytes: &[u8], qap: i32) -> Result<Self, SerializationError> {
        let curve = curve_id::<E::ScalarField>().ok_or_else(|| {
            SerializationError::IoError(ark_std::io::Error::new(ark_std::io::ErrorKind::Other, "libg16b200 does not support this curve"))
        })?;
        let mut ctx = core::ptr::null_mut();
        ser_status(unsafe { sys::g16_ctx_create(curve, device, &mut ctx) })?;
        let mut info = sys::g16_r1cs_info::default();
        let rc = unsafe { sys::g16_r1cs_load(ctx, qap, bytes.as_ptr(), bytes.len() as u64, &mut info) };
        if rc != 0 {
            let err = ser_status(rc);
            unsafe { sys::g16_ctx_destroy(ctx) };
            err?;
        }
        Ok(Self {
            ctx,
            num_inputs: info.num_inputs as usize,
            num_constraints: info.num_constraints as usize,
            num_variables: (info.num_inputs + info.num_witness) as usize,
            fq_limbs: unsafe { sys::g16_fq_limbs(ctx) } as usize,
            g2_limbs: unsafe { sys::g16_g2_limbs(ctx) } as usize,
            flags: Cell::new(0),
            _e: PhantomData,
        })
    }

    /// The proving key of a snarkjs `.zkey` onto the resident circuit (g16_zkey_load with `sys::G16_ZKEY_KEY_ONLY`), which
    /// keeps its C matrix: the circom flow is `load_r1cs(circuit.r1cs, sys::G16_QAP_CIRCOM)` then this with
    /// circuit_final.zkey.  The coefficient section is not read; whether the key belongs to the circuit is
    /// `verify_key`'s question.  Sizes other than the circuit's are `InvalidData` with the previous key kept; a refused point
    /// leaves no key.  Returns the key's VerifyingKey.
    pub fn load_zkey_key(&self, bytes: &[u8], validate: Validate, rank: u32, world: u32) -> Result<VerifyingKey<E>, SerializationError> {
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let (mut alpha_g1, mut beta_g1, mut delta_g1) = (ark_std::vec![0u64; w1], ark_std::vec![0u64; w1], ark_std::vec![0u64; w1]);
        let (mut beta_g2, mut gamma_g2, mut delta_g2) = (ark_std::vec![0u64; w2], ark_std::vec![0u64; w2], ark_std::vec![0u64; w2]);
        let mut abc = ark_std::vec![0u64; w1 * self.num_inputs];
        let null = core::ptr::null_mut();
        let desc = sys::g16_pk_export_desc {
            a_query: null,
            b_g1_query: null,
            b_g2_query: null,
            h_query: null,
            l_query: null,
            alpha_g1: alpha_g1.as_mut_ptr(),
            beta_g1: beta_g1.as_mut_ptr(),
            delta_g1: delta_g1.as_mut_ptr(),
            beta_g2: beta_g2.as_mut_ptr(),
            gamma_g2: gamma_g2.as_mut_ptr(),
            delta_g2: delta_g2.as_mut_ptr(),
            gamma_abc_g1: abc.as_mut_ptr(),
        };
        let flags = sys::G16_ZKEY_KEY_ONLY | if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe {
            sys::g16_zkey_load(self.ctx, bytes.as_ptr(), bytes.len() as u64, flags, rank, world, &desc, core::ptr::null_mut())
        })?;
        Ok(VerifyingKey {
            alpha_g1: unpack_point(&alpha_g1),
            beta_g2: unpack_point(&beta_g2),
            gamma_g2: unpack_point(&gamma_g2),
            delta_g2: unpack_point(&delta_g2),
            gamma_abc_g1: abc.chunks(w1).map(|l| unpack_point(l)).collect(),
        })
    }

    /// The full assignment of a circom / snarkjs `.wtns` (g16_wtns_read: elements checked below r and put in Montgomery form
    /// on the GPU), usable directly as `full_assignment`.  Needs no circuit.  A malformed file or element is `InvalidData`.
    pub fn read_wtns(&self, bytes: &[u8]) -> Result<Vec<E::ScalarField>, SerializationError> {
        let mut n = 0u64;
        ser_status(unsafe { sys::g16_wtns_read(self.ctx, bytes.as_ptr(), bytes.len() as u64, core::ptr::null_mut(), 0, &mut n) })?;
        let mut out = ark_std::vec![E::ScalarField::zero(); n as usize];
        if n > 0 {
            // the ABI's Montgomery limbs are the field elements' memory image
            ser_status(unsafe {
                sys::g16_wtns_read(self.ctx, bytes.as_ptr(), bytes.len() as u64, out.as_mut_ptr() as *mut u64, n, &mut n)
            })?;
        }
        Ok(out)
    }

    /// Replace the resident key by the ark-serialized ProvingKey in `bytes` (g16_pk_load_serialized).  A rejected key
    /// leaves no key resident.
    pub fn load_proving_key_bytes(
        &self,
        bytes: &[u8],
        compress: Compress,
        validate: Validate,
        rank: u32,
        world: u32,
    ) -> Result<VerifyingKey<E>, SerializationError> {
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let (mut alpha_g1, mut beta_g1, mut delta_g1) = (ark_std::vec![0u64; w1], ark_std::vec![0u64; w1], ark_std::vec![0u64; w1]);
        let (mut beta_g2, mut gamma_g2, mut delta_g2) = (ark_std::vec![0u64; w2], ark_std::vec![0u64; w2], ark_std::vec![0u64; w2]);
        let mut abc = ark_std::vec![0u64; w1 * self.num_inputs];
        let null = core::ptr::null_mut();
        let desc = sys::g16_pk_export_desc {
            a_query: null,
            b_g1_query: null,
            b_g2_query: null,
            h_query: null,
            l_query: null,
            alpha_g1: alpha_g1.as_mut_ptr(),
            beta_g1: beta_g1.as_mut_ptr(),
            delta_g1: delta_g1.as_mut_ptr(),
            beta_g2: beta_g2.as_mut_ptr(),
            gamma_g2: gamma_g2.as_mut_ptr(),
            delta_g2: delta_g2.as_mut_ptr(),
            gamma_abc_g1: abc.as_mut_ptr(),
        };
        let mut flags = if matches!(compress, Compress::Yes) { sys::G16_SER_COMPRESSED } else { 0 };
        if matches!(validate, Validate::Yes) {
            flags |= sys::G16_SER_VALIDATE;
        }
        ser_status(unsafe { sys::g16_pk_load_serialized(self.ctx, bytes.as_ptr(), bytes.len() as u64, flags, rank, world, &desc) })?;
        Ok(VerifyingKey {
            alpha_g1: unpack_point(&alpha_g1),
            beta_g2: unpack_point(&beta_g2),
            gamma_g2: unpack_point(&gamma_g2),
            delta_g2: unpack_point(&delta_g2),
            gamma_abc_g1: abc.chunks(w1).map(|l| unpack_point(l)).collect(),
        })
    }

    /// Derives the resident circuit's proving key on the GPU from a powers-of-tau transcript (g16_setup_from_srs) and makes
    /// it resident: gamma = 1, delta = 1 until `contribute_delta`.  `tau_g1` holds at least 2n - 1 points, `tau_g2`,
    /// `alpha_tau_g1` and `beta_tau_g1` at least n (n = the circuit's domain size); longer transcripts are fine.
    /// `validate` adds the subgroup check of every point read.  Export the key with `export_proving_key_bytes`.
    pub fn setup_from_srs(
        &self,
        tau_g1: &[Affine<E::G1Config>],
        tau_g2: &[Affine<E::G2Config>],
        alpha_tau_g1: &[Affine<E::G1Config>],
        beta_tau_g1: &[Affine<E::G1Config>],
        beta_g2: &Affine<E::G2Config>,
        validate: Validate,
    ) -> Result<(), SerializationError> {
        let (t1, t2, a1, b1) = (pack_points(tau_g1), pack_points(tau_g2), pack_points(alpha_tau_g1), pack_points(beta_tau_g1));
        let bg2 = pack_points(core::slice::from_ref(beta_g2));
        let desc = sys::g16_srs_desc {
            tau_g1: t1.as_ptr(),
            tau_g1_len: tau_g1.len() as u64,
            tau_g2: t2.as_ptr(),
            tau_g2_len: tau_g2.len() as u64,
            alpha_tau_g1: a1.as_ptr(),
            alpha_tau_g1_len: alpha_tau_g1.len() as u64,
            beta_tau_g1: b1.as_ptr(),
            beta_tau_g1_len: beta_tau_g1.len() as u64,
            beta_g2: bg2.as_ptr(),
        };
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe { sys::g16_setup_from_srs(self.ctx, &desc, flags) })
    }

    /// A snarkjs `.ptau` powers-of-tau file (g16_ptau_read, copied on the host; every call that takes the points checks
    /// them on the GPU).  With `log_n`, only what a circuit of domain 2^log_n needs: 2n - 1, n, n and n powers and, for a
    /// prepared file, level log_n of its Lagrange points.  Without it, the whole powers and no Lagrange points.  A malformed
    /// file is `InvalidData`; a request the file cannot serve (log_n above its power) is an `IoError` carrying it.
    pub fn read_ptau(&self, bytes: &[u8], log_n: Option<u32>) -> Result<Ptau<E>, SerializationError> {
        let null = core::ptr::null();
        let mut info = sys::g16_ptau_info::default();
        ser_status(unsafe { sys::g16_ptau_read(self.ctx, bytes.as_ptr(), bytes.len() as u64, null, core::ptr::null_mut(), &mut info) })?;
        let np = 1usize << info.power;
        let n = log_n.map_or(np, |k| 1usize << k);
        // below the file's power, the interior H level is checked against and corrected by tau_g1[2n - 1]
        let lens = if log_n.is_some() { [(2 * n).min(2 * np - 1), n, n, n] } else { [2 * np - 1, np, np, np] };
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let (mut t1, mut t2) = (ark_std::vec![0u64; lens[0] * w1], ark_std::vec![0u64; lens[1] * w2]);
        let (mut a1, mut b1, mut bg2) = (ark_std::vec![0u64; lens[2] * w1], ark_std::vec![0u64; lens[3] * w1], ark_std::vec![0u64; w2]);
        let out = sys::g16_srs_out {
            tau_g1: t1.as_mut_ptr(),
            tau_g1_len: lens[0] as u64,
            tau_g2: t2.as_mut_ptr(),
            tau_g2_len: lens[1] as u64,
            alpha_tau_g1: a1.as_mut_ptr(),
            alpha_tau_g1_len: lens[2] as u64,
            beta_tau_g1: b1.as_mut_ptr(),
            beta_tau_g1_len: lens[3] as u64,
            beta_g2: bg2.as_mut_ptr(),
        };
        let lag = log_n.filter(|_| info.prepared != 0);
        let (mut l1, mut l2, mut la, mut lb, mut lh) = if lag.is_some() {
            (ark_std::vec![0u64; n * w1], ark_std::vec![0u64; n * w2], ark_std::vec![0u64; n * w1], ark_std::vec![0u64; n * w1], ark_std::vec![0u64; n * w1])
        } else {
            (Vec::new(), Vec::new(), Vec::new(), Vec::new(), Vec::new())
        };
        let mut lout = sys::g16_lagrange_out {
            log_n: lag.unwrap_or(0),
            h_over_2n: 0,
            tau_g1: l1.as_mut_ptr(),
            tau_g2: l2.as_mut_ptr(),
            alpha_tau_g1: la.as_mut_ptr(),
            beta_tau_g1: lb.as_mut_ptr(),
            tau_g1_h: lh.as_mut_ptr(),
        };
        let lptr = if lag.is_some() { &mut lout as *mut sys::g16_lagrange_out } else { core::ptr::null_mut() };
        ser_status(unsafe { sys::g16_ptau_read(self.ctx, bytes.as_ptr(), bytes.len() as u64, &out, lptr, &mut info) })?;
        fn points<P: SWCurveConfig>(v: &[u64]) -> Vec<Affine<P>> {
            v.chunks(point_limbs::<P>()).map(|l| unpack_point(l)).collect()
        }
        Ok(Ptau {
            power: info.power,
            ceremony_power: info.ceremony_power,
            prepared: info.prepared != 0,
            srs: PowersOfTau {
                tau_g1: points(&t1),
                tau_g2: points(&t2),
                alpha_tau_g1: points(&a1),
                beta_tau_g1: points(&b1),
                beta_g2: unpack_point(&bg2),
            },
            lagrange: lag.map(|k| LagrangePoints {
                log_n: k,
                h_over_2n: lout.h_over_2n != 0,
                tau_g1: points(&l1),
                tau_g2: points(&l2),
                alpha_tau_g1: points(&la),
                beta_tau_g1: points(&lb),
                tau_g1_h: points(&lh),
            }),
        })
    }

    /// Derives the resident circuit's proving key from a transcript and one level of its Lagrange points
    /// (g16_setup_from_lagrange): the key `setup_from_srs` makes from `srs`, limb for limb, without the group transforms.
    /// The points are first checked against `srs` on the GPU under the challenge `rho` (draw it after the file is fixed);
    /// a member that is not the transform of the transcript, or a refused point, is `InvalidData` and leaves no key.
    /// `validate` adds the subgroup check of every point, without which the check means nothing on a curve whose cofactor
    /// is not 1.
    pub fn setup_from_lagrange(
        &self,
        srs: &PowersOfTau<E>,
        lag: &LagrangePoints<E>,
        rho: E::ScalarField,
        validate: Validate,
    ) -> Result<(), SerializationError> {
        let (t1, t2, a1, b1) =
            (pack_points(&srs.tau_g1), pack_points(&srs.tau_g2), pack_points(&srs.alpha_tau_g1), pack_points(&srs.beta_tau_g1));
        let bg2 = pack_points(core::slice::from_ref(&srs.beta_g2));
        let desc = sys::g16_srs_desc {
            tau_g1: t1.as_ptr(),
            tau_g1_len: srs.tau_g1.len() as u64,
            tau_g2: t2.as_ptr(),
            tau_g2_len: srs.tau_g2.len() as u64,
            alpha_tau_g1: a1.as_ptr(),
            alpha_tau_g1_len: srs.alpha_tau_g1.len() as u64,
            beta_tau_g1: b1.as_ptr(),
            beta_tau_g1_len: srs.beta_tau_g1.len() as u64,
            beta_g2: bg2.as_ptr(),
        };
        let (l1, l2, la, lb, lh) = (
            pack_points(&lag.tau_g1),
            pack_points(&lag.tau_g2),
            pack_points(&lag.alpha_tau_g1),
            pack_points(&lag.beta_tau_g1),
            pack_points(&lag.tau_g1_h),
        );
        let ptr = |v: &Vec<u64>| if v.is_empty() { core::ptr::null() } else { v.as_ptr() };
        let ldesc = sys::g16_lagrange_desc {
            log_n: lag.log_n,
            h_over_2n: lag.h_over_2n as u32,
            tau_g1: ptr(&l1),
            tau_g2: ptr(&l2),
            alpha_tau_g1: ptr(&la),
            beta_tau_g1: ptr(&lb),
            tau_g1_h: ptr(&lh),
        };
        let r = [rho];
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe { sys::g16_setup_from_lagrange(self.ctx, &desc, &ldesc, scalars_ptr(&r), flags) })
    }

    /// The resident circuit's proving key from a snarkjs `.ptau` file: `read_ptau` for the circuit's domain, then
    /// `setup_from_lagrange` (challenge drawn from `rng`) when the file is prepared and `setup_from_srs` when it is not.
    /// Both give the same key: gamma = 1, delta = 1 until `contribute_delta`.
    pub fn setup_from_ptau<R: RngCore>(&self, bytes: &[u8], rng: &mut R, validate: Validate) -> Result<(), SerializationError> {
        let log_n = unsafe { sys::g16_domain_log(self.ctx) };
        let p = self.read_ptau(bytes, Some(log_n))?;
        match &p.lagrange {
            Some(lag) => {
                let rho = loop {
                    let x = E::ScalarField::rand(rng);
                    if !x.is_zero() {
                        break x;
                    }
                };
                self.setup_from_lagrange(&p.srs, lag, rho, validate)
            }
            None => self.setup_from_srs(&p.srs.tau_g1, &p.srs.tau_g2, &p.srs.alpha_tau_g1, &p.srs.beta_tau_g1, &p.srs.beta_g2, validate),
        }
    }

    /// One phase-1 contribution (g16_srs_contribute, snarkjs `powersoftau contribute`) to a powers-of-tau transcript, on the
    /// GPU: point i of `tau_g1` and `tau_g2` times tau^i, of `alpha_tau_g1` times alpha tau^i, of `beta_tau_g1` times
    /// beta tau^i, and `beta_g2` times beta.  Members may have any length below 2^32 and may be empty.  `validate` adds the
    /// subgroup check of every point; `chunk_points` caps the points per chunk (0: as many as the free device memory holds).
    /// A refused point is `InvalidData` (the message naming member and index goes to stderr); a zero secret is an `IoError`
    /// carrying "UnexpectedIdentity".  Needs no circuit or key and leaves the resident ones alone.
    #[allow(clippy::too_many_arguments)]
    pub fn contribute_srs(
        &self,
        tau_g1: &[Affine<E::G1Config>],
        tau_g2: &[Affine<E::G2Config>],
        alpha_tau_g1: &[Affine<E::G1Config>],
        beta_tau_g1: &[Affine<E::G1Config>],
        beta_g2: &Affine<E::G2Config>,
        tau: E::ScalarField,
        alpha: E::ScalarField,
        beta: E::ScalarField,
        validate: Validate,
        chunk_points: u64,
    ) -> Result<PowersOfTau<E>, SerializationError> {
        // packed copies, transformed in place by the library
        let (mut t1, mut t2, mut a1, mut b1) =
            (pack_points(tau_g1), pack_points(tau_g2), pack_points(alpha_tau_g1), pack_points(beta_tau_g1));
        let mut bg2 = pack_points(core::slice::from_ref(beta_g2));
        let desc = sys::g16_srs_desc {
            tau_g1: t1.as_ptr(),
            tau_g1_len: tau_g1.len() as u64,
            tau_g2: t2.as_ptr(),
            tau_g2_len: tau_g2.len() as u64,
            alpha_tau_g1: a1.as_ptr(),
            alpha_tau_g1_len: alpha_tau_g1.len() as u64,
            beta_tau_g1: b1.as_ptr(),
            beta_tau_g1_len: beta_tau_g1.len() as u64,
            beta_g2: bg2.as_ptr(),
        };
        let out = sys::g16_srs_out {
            tau_g1: t1.as_mut_ptr(),
            tau_g1_len: tau_g1.len() as u64,
            tau_g2: t2.as_mut_ptr(),
            tau_g2_len: tau_g2.len() as u64,
            alpha_tau_g1: a1.as_mut_ptr(),
            alpha_tau_g1_len: alpha_tau_g1.len() as u64,
            beta_tau_g1: b1.as_mut_ptr(),
            beta_tau_g1_len: beta_tau_g1.len() as u64,
            beta_g2: bg2.as_mut_ptr(),
        };
        let (t, a, b) = ([tau], [alpha], [beta]);
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe {
            sys::g16_srs_contribute(self.ctx, &desc, scalars_ptr(&t), scalars_ptr(&a), scalars_ptr(&b), flags, chunk_points, &out)
        })?;
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        Ok(PowersOfTau {
            tau_g1: t1.chunks(w1).map(|l| unpack_point(l)).collect(),
            tau_g2: t2.chunks(w2).map(|l| unpack_point(l)).collect(),
            alpha_tau_g1: a1.chunks(w1).map(|l| unpack_point(l)).collect(),
            beta_tau_g1: b1.chunks(w1).map(|l| unpack_point(l)).collect(),
            beta_g2: unpack_point(&bg2),
        })
    }

    /// The GPU part of checking a powers-of-tau transcript (g16_srs_verify_pairs, snarkjs `powersoftau verify` without the
    /// proofs of knowledge, which are `contribution_chain_pairs`): every point is checked (curve, with `validate` the subgroup,
    /// never the identity), tau_g1[0] must
    /// be `g1` and tau_g2[0] must be `g2`, and one MSM per member under the challenge `rho` (non-zero, drawn after the
    /// transcript is fixed) reduces each member's chain to one pairing equation.  Returns the five equations as
    /// (P, Q, P', Q'); equation k holds iff e(P, Q) = e(P', Q').  A refused point is `InvalidData` (the message naming
    /// member and index goes to stderr); an argument error (a member too short, rho = 0) is an `IoError` carrying it.
    #[allow(clippy::type_complexity)]
    pub fn srs_verification_pairs(
        &self,
        srs: &PowersOfTau<E>,
        g1: &Affine<E::G1Config>,
        g2: &Affine<E::G2Config>,
        rho: E::ScalarField,
        validate: Validate,
        chunk_points: u64,
    ) -> Result<[(Affine<E::G1Config>, Affine<E::G2Config>, Affine<E::G1Config>, Affine<E::G2Config>); 5], SerializationError>
    {
        let (t1, t2, a1, b1) =
            (pack_points(&srs.tau_g1), pack_points(&srs.tau_g2), pack_points(&srs.alpha_tau_g1), pack_points(&srs.beta_tau_g1));
        let bg2 = pack_points(core::slice::from_ref(&srs.beta_g2));
        let desc = sys::g16_srs_desc {
            tau_g1: t1.as_ptr(),
            tau_g1_len: srs.tau_g1.len() as u64,
            tau_g2: t2.as_ptr(),
            tau_g2_len: srs.tau_g2.len() as u64,
            alpha_tau_g1: a1.as_ptr(),
            alpha_tau_g1_len: srs.alpha_tau_g1.len() as u64,
            beta_tau_g1: b1.as_ptr(),
            beta_tau_g1_len: srs.beta_tau_g1.len() as u64,
            beta_g2: bg2.as_ptr(),
        };
        let (gp1, gp2) = (pack_points(core::slice::from_ref(g1)), pack_points(core::slice::from_ref(g2)));
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let (mut o1, mut o2) = (vec![0u64; 10 * w1], vec![0u64; 10 * w2]);
        let r = [rho];
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe {
            sys::g16_srs_verify_pairs(
                self.ctx,
                &desc,
                gp1.as_ptr(),
                gp2.as_ptr(),
                scalars_ptr(&r),
                flags,
                chunk_points,
                o1.as_mut_ptr(),
                o2.as_mut_ptr(),
            )
        })?;
        let p = |i: usize| unpack_point::<E::G1Config>(&o1[i * w1..(i + 1) * w1]);
        let q = |i: usize| unpack_point::<E::G2Config>(&o2[i * w2..(i + 1) * w2]);
        Ok(core::array::from_fn(|k| (p(2 * k), q(2 * k), p(2 * k + 1), q(2 * k + 1))))
    }

    /// Checks a powers-of-tau transcript over the generators `g1`, `g2`: `srs_verification_pairs` under a challenge drawn
    /// from `rng`, then each equation as `E::multi_pairing([P, -P'], [Q, Q']).is_zero()`.  Ok(true): with probability at
    /// least 1 - N/r the transcript is T(tau, alpha, beta) for non-zero tau, alpha, beta with one tau in both groups.
    /// Ok(false): an equation fails.  A point the library refuses (off the curve, outside the subgroup with `validate`,
    /// the identity, a wrong generator) is `InvalidData`.  `validate` should be `Yes` unless the points were checked
    /// already: without it the answer means nothing on a curve whose cofactor is not 1.
    pub fn verify_srs<R: RngCore>(
        &self,
        srs: &PowersOfTau<E>,
        g1: &Affine<E::G1Config>,
        g2: &Affine<E::G2Config>,
        rng: &mut R,
        validate: Validate,
        chunk_points: u64,
    ) -> Result<bool, SerializationError> {
        let rho = loop {
            let x = E::ScalarField::rand(rng);
            if !x.is_zero() {
                break x;
            }
        };
        let eqs = self.srs_verification_pairs(srs, g1, g2, rho, validate, chunk_points)?;
        Ok(eqs.iter().all(|(p, q, p2, q2)| E::multi_pairing([*p, -*p2], [*q, *q2]).is_zero()))
    }

    /// The GPU part of checking that `pk` is the key of the resident circuit made from the transcript `srs`
    /// (g16_pk_verify_pairs, snarkjs `zkey verify`; the contributions' proofs of knowledge are `contribution_chain_pairs`).
    /// The library checks every point (curve, with `validate` the subgroup), that alpha_g1, beta_g1 and beta_g2 are the
    /// transcript's, that delta and gamma are not the identity, that gamma_g2 != delta_g2 (`uncontributed` accepts the initial key of a ceremony, where
    /// gamma = delta = 1), and that the random combinations of a_query, b_g1_query and b_g2_query under the challenge `rho`
    /// match the transcript's.  Returns the four equations (delta, h_query, l_query, gamma_abc_g1) as (P, Q, P', Q');
    /// equation k holds iff e(P, Q) = e(P', Q').  A refusal is `InvalidData` (the message naming the member goes to
    /// stderr); an argument error (a transcript too short for the circuit, rho = 0) is an `IoError` carrying it.
    #[allow(clippy::type_complexity)]
    pub fn key_verification_pairs(
        &self,
        pk: &ProvingKey<E>,
        srs: &PowersOfTau<E>,
        rho: E::ScalarField,
        validate: Validate,
        uncontributed: bool,
    ) -> Result<[(Affine<E::G1Config>, Affine<E::G2Config>, Affine<E::G1Config>, Affine<E::G2Config>); 4], SerializationError>
    {
        let (t1, t2, a1, b1) =
            (pack_points(&srs.tau_g1), pack_points(&srs.tau_g2), pack_points(&srs.alpha_tau_g1), pack_points(&srs.beta_tau_g1));
        let bg2 = pack_points(core::slice::from_ref(&srs.beta_g2));
        let sdesc = sys::g16_srs_desc {
            tau_g1: t1.as_ptr(),
            tau_g1_len: srs.tau_g1.len() as u64,
            tau_g2: t2.as_ptr(),
            tau_g2_len: srs.tau_g2.len() as u64,
            alpha_tau_g1: a1.as_ptr(),
            alpha_tau_g1_len: srs.alpha_tau_g1.len() as u64,
            beta_tau_g1: b1.as_ptr(),
            beta_tau_g1_len: srs.beta_tau_g1.len() as u64,
            beta_g2: bg2.as_ptr(),
        };
        let (aq, bq1, bq2, hq, lq, abc) = (
            pack_points(&pk.a_query),
            pack_points(&pk.b_g1_query),
            pack_points(&pk.b_g2_query),
            pack_points(&pk.h_query),
            pack_points(&pk.l_query),
            pack_points(&pk.vk.gamma_abc_g1),
        );
        let (alpha_g1, beta_g1, delta_g1) =
            (pack_points(&[pk.vk.alpha_g1]), pack_points(&[pk.beta_g1]), pack_points(&[pk.delta_g1]));
        let (beta_g2, gamma_g2, delta_g2) =
            (pack_points(&[pk.vk.beta_g2]), pack_points(&[pk.vk.gamma_g2]), pack_points(&[pk.vk.delta_g2]));
        let kdesc = sys::g16_pk_check_desc {
            a_query: aq.as_ptr(),
            b_g1_query: bq1.as_ptr(),
            b_g2_query: bq2.as_ptr(),
            h_query: hq.as_ptr(),
            l_query: lq.as_ptr(),
            alpha_g1: alpha_g1.as_ptr(),
            beta_g1: beta_g1.as_ptr(),
            delta_g1: delta_g1.as_ptr(),
            beta_g2: beta_g2.as_ptr(),
            gamma_g2: gamma_g2.as_ptr(),
            delta_g2: delta_g2.as_ptr(),
            gamma_abc_g1: abc.as_ptr(),
        };
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let (mut o1, mut o2) = (vec![0u64; 8 * w1], vec![0u64; 8 * w2]);
        let r = [rho];
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 }
            | if uncontributed { sys::G16_PK_UNCONTRIBUTED } else { 0 };
        ser_status(unsafe {
            sys::g16_pk_verify_pairs(self.ctx, &sdesc, &kdesc, scalars_ptr(&r), flags, o1.as_mut_ptr(), o2.as_mut_ptr())
        })?;
        let p = |i: usize| unpack_point::<E::G1Config>(&o1[i * w1..(i + 1) * w1]);
        let q = |i: usize| unpack_point::<E::G2Config>(&o2[i * w2..(i + 1) * w2]);
        Ok(core::array::from_fn(|k| (p(2 * k), q(2 * k), p(2 * k + 1), q(2 * k + 1))))
    }

    /// Checks that `pk` is the key of the resident circuit made from the transcript `srs`: `key_verification_pairs` under a
    /// challenge drawn from `rng` (with `validate` = Yes and no uncontributed key), then each equation as
    /// `E::multi_pairing([P, -P'], [Q, Q']).is_zero()`.  Ok(true): with probability at least 1 - 6 max(nv, n) / r the key is
    /// the setup of the transcript's tau, alpha, beta with some gamma != delta.  Ok(false): an equation fails.  A key the
    /// library refuses itself is `InvalidData`.  The transcript should have passed `verify_srs` first.
    pub fn verify_key<R: RngCore>(&self, pk: &ProvingKey<E>, srs: &PowersOfTau<E>, rng: &mut R) -> Result<bool, SerializationError> {
        let rho = loop {
            let x = E::ScalarField::rand(rng);
            if !x.is_zero() {
                break x;
            }
        };
        let eqs = self.key_verification_pairs(pk, srs, rho, Validate::Yes, false)?;
        Ok(eqs.iter().all(|(p, q, p2, q2)| E::multi_pairing([*p, -*p2], [*q, *q2]).is_zero()))
    }

    /// One phase-2 contribution to the resident key (g16_setup_contribute): delta_g1, delta_g2 times `delta`, the H and L
    /// queries times delta^-1.  delta = 0 is SynthesisError::UnexpectedIdentity.
    pub fn contribute_delta(&self, delta: E::ScalarField) -> R1CSResult<()> {
        if delta.is_zero() {
            return Err(SynthesisError::UnexpectedIdentity);
        }
        let d = [delta];
        status(unsafe { sys::g16_setup_contribute(self.ctx, scalars_ptr(&d)) })
    }

    /// One phase-2 contribution to a key received from another party (g16_pk_contribute, snarkjs `zkey contribute`):
    /// delta_g1 and delta_g2 times `delta`, every h_query and l_query point times delta^-1 on the GPU, in chunks of at most
    /// `chunk_points` points (0: as many as the device memory holds).  Every other member is copied from `pk`.  Every point is
    /// checked first (curve, with `validate` the subgroup; delta_g1 and delta_g2 not the identity): a refused point is
    /// `InvalidData` (the message naming member and index goes to stderr).  delta = 0 is an `IoError` carrying
    /// "UnexpectedIdentity".  Needs no circuit or key and leaves the resident ones alone.
    pub fn contribute_key(
        &self,
        pk: &ProvingKey<E>,
        delta: E::ScalarField,
        validate: Validate,
        chunk_points: u64,
    ) -> Result<ProvingKey<E>, SerializationError> {
        // packed copies, transformed in place by the library
        let (mut hq, mut lq) = (pack_points(&pk.h_query), pack_points(&pk.l_query));
        let (mut d1, mut d2) = (pack_points(&[pk.delta_g1]), pack_points(&[pk.vk.delta_g2]));
        let desc = sys::g16_pk_delta_desc {
            h_query: hq.as_ptr(),
            h_len: pk.h_query.len() as u64,
            l_query: lq.as_ptr(),
            l_len: pk.l_query.len() as u64,
            delta_g1: d1.as_ptr(),
            delta_g2: d2.as_ptr(),
        };
        let out = sys::g16_pk_delta_out {
            h_query: hq.as_mut_ptr(),
            h_len: pk.h_query.len() as u64,
            l_query: lq.as_mut_ptr(),
            l_len: pk.l_query.len() as u64,
            delta_g1: d1.as_mut_ptr(),
            delta_g2: d2.as_mut_ptr(),
        };
        let d = [delta];
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe { sys::g16_pk_contribute(self.ctx, &desc, scalars_ptr(&d), flags, chunk_points, &out) })?;
        let w1 = point_limbs::<E::G1Config>();
        let mut key = pk.clone();
        key.h_query = hq.chunks(w1).map(|l| unpack_point(l)).collect();
        key.l_query = lq.chunks(w1).map(|l| unpack_point(l)).collect();
        key.delta_g1 = unpack_point(&d1);
        key.vk.delta_g2 = unpack_point(&d2);
        Ok(key)
    }

    /// The proofs of knowledge of a chain of contributions (g16_contribution_chain_pairs), phase 1 or phase 2: from the
    /// running point `start` (phase 2: the uncontributed key's delta_g1 = tau_g1[0]) to `end` (the final key's delta_g1)
    /// through `records`.  The library checks every point (curve, with `validate` the subgroup, never the identity) and that
    /// the last record ends at `end`; a refusal is `InvalidData` (the message naming record and member goes to stderr).
    /// Returns 2 records.len() equations as (P, Q, P', Q'), equation k holding iff e(P, Q) = e(P', Q'): 2i is record i's
    /// proof of knowledge (s, r_x) = (s_x, r), 2i + 1 its step (D_i, r_x) = (D_(i+1), r).  Each record's `r_g2` must have
    /// been recomputed by the caller from the ceremony's transcript.
    #[allow(clippy::type_complexity)]
    pub fn contribution_chain_pairs(
        &self,
        start: &Affine<E::G1Config>,
        end: &Affine<E::G1Config>,
        records: &[ContributionRecord<E>],
        validate: Validate,
    ) -> Result<Vec<(Affine<E::G1Config>, Affine<E::G2Config>, Affine<E::G1Config>, Affine<E::G2Config>)>, SerializationError> {
        let (sp, ep) = (pack_points(core::slice::from_ref(start)), pack_points(core::slice::from_ref(end)));
        let packed: Vec<[Vec<u64>; 5]> = records
            .iter()
            .map(|c| {
                [
                    pack_points(&[c.after_g1]),
                    pack_points(&[c.s_g1]),
                    pack_points(&[c.s_x_g1]),
                    pack_points(&[c.r_g2]),
                    pack_points(&[c.r_x_g2]),
                ]
            })
            .collect();
        let descs: Vec<sys::g16_contribution_record> = packed
            .iter()
            .map(|p| sys::g16_contribution_record {
                after_g1: p[0].as_ptr(),
                s_g1: p[1].as_ptr(),
                s_x_g1: p[2].as_ptr(),
                r_g2: p[3].as_ptr(),
                r_x_g2: p[4].as_ptr(),
            })
            .collect();
        let (w1, w2) = (point_limbs::<E::G1Config>(), point_limbs::<E::G2Config>());
        let n = 4 * records.len();
        let (mut o1, mut o2) = (vec![0u64; n * w1], vec![0u64; n * w2]);
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        ser_status(unsafe {
            sys::g16_contribution_chain_pairs(
                self.ctx,
                sp.as_ptr(),
                ep.as_ptr(),
                descs.as_ptr(),
                records.len() as u32,
                flags,
                o1.as_mut_ptr(),
                o2.as_mut_ptr(),
            )
        })?;
        let p = |i: usize| unpack_point::<E::G1Config>(&o1[i * w1..(i + 1) * w1]);
        let q = |i: usize| unpack_point::<E::G2Config>(&o2[i * w2..(i + 1) * w2]);
        Ok((0..2 * records.len()).map(|k| (p(2 * k), q(2 * k), p(2 * k + 1), q(2 * k + 1))).collect())
    }

    /// Checks a chain of contributions: `contribution_chain_pairs` with `validate` = Yes, then each equation as
    /// `E::multi_pairing([P, -P'], [Q, Q']).is_zero()`.  Ok(true): end = (prod x_i) start, and contributor i knew x_i when
    /// its r_g2 is a random-oracle output over its contribution's transcript, so one honest contributor makes the product
    /// unknown.  Ok(false): an equation fails.  In phase 2, run it from tau_g1[0] to the final key's delta_g1 together with
    /// `verify_key` on the final key.
    pub fn verify_contribution_chain(
        &self,
        start: &Affine<E::G1Config>,
        end: &Affine<E::G1Config>,
        records: &[ContributionRecord<E>],
    ) -> Result<bool, SerializationError> {
        let eqs = self.contribution_chain_pairs(start, end, records, Validate::Yes)?;
        Ok(eqs.iter().all(|(p, q, p2, q2)| E::multi_pairing([*p, -*p2], [*q, *q2]).is_zero()))
    }

    /// snarkjs `powersoftau prepare phase2` on the GPU (g16_ptau_prepare): the `.ptau` file `bytes` with its Lagrange
    /// sections 12..15 computed from the powers (those of a prepared input are recomputed).  Every point of sections 2..5 is
    /// checked first, with `Validate::Yes` also in the prime-order subgroup; a refused point is `InvalidData`, the message
    /// naming it.  The file is not checked to be a powers-of-tau transcript (`verify_srs` does that).
    pub fn prepare_ptau(&self, bytes: &[u8], validate: Validate) -> Result<Vec<u8>, SerializationError> {
        let flags = if matches!(validate, Validate::Yes) { sys::G16_SER_VALIDATE } else { 0 };
        let mut n = 0u64;
        ser_status(unsafe { sys::g16_ptau_prepare(self.ctx, bytes.as_ptr(), bytes.len() as u64, flags, core::ptr::null_mut(), 0, &mut n) })?;
        let mut out = ark_std::vec![0u8; n as usize];
        ser_status(unsafe { sys::g16_ptau_prepare(self.ctx, bytes.as_ptr(), bytes.len() as u64, flags, out.as_mut_ptr(), n, &mut n) })?;
        Ok(out)
    }

    /// `ProvingKey::serialize_with_mode(compress)` of the resident key, encoded on the GPU (g16_pk_export_serialized).  Only
    /// a key made by the library's own setup can be exported.
    pub fn export_proving_key_bytes(&self, compress: Compress) -> Result<Vec<u8>, SerializationError> {
        let flags = if matches!(compress, Compress::Yes) { sys::G16_SER_COMPRESSED } else { 0 };
        let mut n = 0u64;
        ser_status(unsafe { sys::g16_pk_export_serialized(self.ctx, flags, core::ptr::null_mut(), 0, &mut n) })?;
        let mut out = ark_std::vec![0u8; n as usize];
        ser_status(unsafe { sys::g16_pk_export_serialized(self.ctx, flags, out.as_mut_ptr(), n, &mut n) })?;
        Ok(out)
    }

    /// a (G1) || b (G2) || c (G1): 8 * fq_limbs, or 6 * fq_limbs on BW6-761
    fn proof_limbs(&self) -> usize {
        4 * self.fq_limbs + self.g2_limbs
    }
    fn proof_from_limbs(&self, out: &[u64]) -> Proof<E> {
        let (n, g) = (self.fq_limbs, self.g2_limbs);
        Proof { a: unpack_point(&out[..2 * n]), b: unpack_point(&out[2 * n..2 * n + g]), c: unpack_point(&out[2 * n + g..4 * n + g]) }
    }

    /// Check every assignment against the circuit on the GPU before proving it (`G16_CHECK_WITNESS` on every prove call of
    /// this prover).  Off by default.  A refused proof is `SynthesisError::Unsatisfiable`, with the constraint or element
    /// on stderr; in `create_proofs_batch` the whole call fails (`check_witness` tells which assignments were bad).
    pub fn set_check_witness(&self, on: bool) {
        let f = self.flags.get() & !sys::G16_CHECK_WITNESS;
        self.flags.set(if on { f | sys::G16_CHECK_WITNESS } else { f });
    }

    /// g16_check_witness: one report per assignment (fields as in the header; `sys::G16_NONE` where there is none).
    pub fn check_witness(&self, assignments: &[Vec<E::ScalarField>]) -> R1CSResult<Vec<sys::g16_witness_report>> {
        if assignments.iter().any(|z| z.len() != self.num_variables) || assignments.len() > u32::MAX as usize {
            return Err(SynthesisError::MalformedVerifyingKey);
        }
        let mut out = ark_std::vec![sys::g16_witness_report::default(); assignments.len()];
        if assignments.is_empty() {
            return Ok(out);
        }
        let z: Vec<E::ScalarField> = assignments.concat();
        status(unsafe { sys::g16_check_witness(self.ctx, assignments.len() as u32, scalars_ptr(&z), 0, out.as_mut_ptr()) })?;
        Ok(out)
    }
    fn check_one(&self, full_assignment: &[E::ScalarField]) -> R1CSResult<sys::g16_witness_report> {
        if full_assignment.len() != self.num_variables {
            return Err(SynthesisError::MalformedVerifyingKey);
        }
        let mut w = sys::g16_witness_report::default();
        status(unsafe { sys::g16_check_witness(self.ctx, 1, scalars_ptr(full_assignment), 0, &mut w) })?;
        Ok(w)
    }
    /// `ConstraintSystem::is_satisfied` of `full_assignment` (instance || witness) on the resident circuit.  An element that
    /// is not a canonical field element, or a first element other than One, is unsatisfied.
    pub fn is_satisfied(&self, full_assignment: &[E::ScalarField]) -> R1CSResult<bool> {
        let w = self.check_one(full_assignment)?;
        Ok(w.first_malformed == sys::G16_NONE && w.num_unsatisfied == 0)
    }
    /// `ConstraintSystem::which_is_unsatisfied`, by index: the lowest unsatisfied constraint (there are no constraint
    /// names at this boundary).  A malformed assignment is `SynthesisError::Unsatisfiable`.
    pub fn which_is_unsatisfied(&self, full_assignment: &[E::ScalarField]) -> R1CSResult<Option<usize>> {
        let w = self.check_one(full_assignment)?;
        if w.first_malformed != sys::G16_NONE {
            eprintln!("libg16b200: assignment element {} is malformed", w.first_malformed);
            return Err(SynthesisError::Unsatisfiable);
        }
        Ok(if w.first_unsatisfied == sys::G16_NONE { None } else { Some(w.first_unsatisfied as usize) })
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
        let mut out = ark_std::vec![0u64; self.proof_limbs()];
        status(unsafe {
            sys::g16_prove(self.ctx, fp_limbs(&r).as_ptr(), fp_limbs(&s).as_ptr(), scalars_ptr(full_assignment), self.flags.get(), out.as_mut_ptr())
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

    /// Many proofs of the resident circuit in one call (g16_prove_batch; no reference counterpart).  Proof i equals
    /// `create_proof_with_reduction_and_matrices` with (rs[i], ss[i], assignments[i]).
    pub fn create_proofs_batch(
        &self,
        rs: &[E::ScalarField],
        ss: &[E::ScalarField],
        assignments: &[Vec<E::ScalarField>],
    ) -> R1CSResult<Vec<Proof<E>>> {
        let count = assignments.len();
        if rs.len() != count || ss.len() != count || assignments.iter().any(|z| z.len() != self.num_variables) {
            return Err(SynthesisError::MalformedVerifyingKey);
        }
        if count == 0 {
            return Ok(Vec::new());
        }
        let z: Vec<E::ScalarField> = assignments.concat();
        let w = self.proof_limbs();
        let mut out = ark_std::vec![0u64; count * w];
        status(unsafe {
            sys::g16_prove_batch(self.ctx, count as u32, scalars_ptr(rs), scalars_ptr(ss), scalars_ptr(&z), 0, self.flags.get(), out.as_mut_ptr())
        })?;
        Ok(out.chunks(w).map(|p| self.proof_from_limbs(p)).collect())
    }
    /// `create_proofs_batch` with fresh randomness: for each proof `r` is sampled before `s`, as src/prover.rs:146-147.
    pub fn create_random_proofs_batch(&self, assignments: &[Vec<E::ScalarField>], rng: &mut impl Rng) -> R1CSResult<Vec<Proof<E>>> {
        let mut rs = Vec::with_capacity(assignments.len());
        let mut ss = Vec::with_capacity(assignments.len());
        for _ in assignments {
            rs.push(E::ScalarField::rand(rng));
            ss.push(E::ScalarField::rand(rng));
        }
        self.create_proofs_batch(&rs, &ss, assignments)
    }

    /// Multi-GPU, first half: this rank's five partial MSM sums ([h, l, a, b_g1] G1 affine, then b_g2 G2 affine).
    pub fn prove_partial(&self, r: E::ScalarField, full_assignment: &[E::ScalarField]) -> R1CSResult<Vec<u64>> {
        let mut out = ark_std::vec![0u64; unsafe { sys::g16_partial_limbs(self.ctx) } as usize];
        status(unsafe { sys::g16_prove_partial(self.ctx, fp_limbs(&r).as_ptr(), scalars_ptr(full_assignment), self.flags.get(), out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Multi-GPU, second half: all ranks' partial records (rank order), gathered by the caller (MPI / NCCL all-gather).
    pub fn prove_assemble(&self, r: E::ScalarField, s: E::ScalarField, partials: &[u64], nparts: u32) -> R1CSResult<Proof<E>> {
        let mut out = ark_std::vec![0u64; self.proof_limbs()];
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
    // (reduction, instance vars, witness vars, constraints, nnz(a)) of the resident circuit: a circuit loaded under one
    // reduction is never reused for the other
    loaded: Option<(i32, usize, usize, usize, usize)>,
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
fn load_matrices_once<F: PrimeField>(t: &mut ThreadCtx, m: &ConstraintMatrices<F>, qap: i32) -> R1CSResult<()> {
    let key = (qap, m.num_instance_variables, m.num_witness_variables, m.num_constraints, m.a_num_non_zero);
    if t.loaded == Some(key) {
        return Ok(());
    }
    t.loaded = None; // a failed load below may have replaced part of the resident circuit
    let (a, b, c) = (Csr::new(&m.a), Csr::new(&m.b), Csr::new(&m.c));
    status(unsafe {
        sys::g16_circuit_load_qap(
            t.ctx,
            qap,
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

/// g16_witness_map on this thread's context with `matrices` resident under the reduction `qap`: n values (LibsnarkReduction:
/// coefficients of h; CircomReduction: evaluations at the odd powers of omega_2n)
fn gpu_witness_map<F: PrimeField>(
    matrices: &ConstraintMatrices<F>,
    num_inputs: usize,
    num_constraints: usize,
    full_assignment: &[F],
    qap: i32,
) -> R1CSResult<Vec<F>> {
    with_thread_ctx::<F, _>(|t| {
        load_matrices_once(t, matrices, qap)?;
        let n = (num_constraints + num_inputs).next_power_of_two();
        let mut h = ark_std::vec![F::zero(); n];
        status(unsafe { sys::g16_witness_map(t.ctx, scalars_ptr(full_assignment), 0, h.as_mut_ptr() as *mut u64) })?;
        Ok(h)
    })
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
        gpu_witness_map(matrices, num_inputs, num_constraints, full_assignment, sys::G16_QAP_LIBSNARK)
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
// ark-circom's CircomReduction with its witness map on the GPU: `ark_groth16::Groth16<E, GpuCircomReduction>` makes and
// uses the same keys and proofs as `Groth16<E, ark_circom::CircomReduction>`.  ark-circom is not a dependency of this
// crate; the reduction is restated from its definition:
//   witness map: c = a o b (matrix C is not read); a, b, c interpolated on the domain of size n and evaluated at the odd
//                powers omega_2n^(2j+1); h[j] = A[j] B[j] - C[j] (n evaluations)
//   H query:     the odd entries of the size-2n ifft of delta^-1 t^i (i < 2n - 1; entry 2n - 1 is zero): n scalars
// ---------------------------------------------------------------------------------------------------------------------
pub struct GpuCircomReduction;

impl R1CSToQAP for GpuCircomReduction {
    fn instance_map_with_evaluation<F: PrimeField, D: EvaluationDomain<F>>(
        cs: ConstraintSystemRef<F>,
        t: &F,
    ) -> Result<(Vec<F>, Vec<F>, Vec<F>, F, usize, usize), SynthesisError> {
        LibsnarkReduction::instance_map_with_evaluation::<F, D>(cs, t) // CircomReduction's is LibsnarkReduction's
    }

    fn witness_map_from_matrices<F: PrimeField, D: EvaluationDomain<F>>(
        matrices: &ConstraintMatrices<F>,
        num_inputs: usize,
        num_constraints: usize,
        full_assignment: &[F],
    ) -> R1CSResult<Vec<F>> {
        gpu_witness_map(matrices, num_inputs, num_constraints, full_assignment, sys::G16_QAP_CIRCOM)
    }

    /// max_power = n - 1 (generator.rs passes the domain size minus one); zt is not used
    fn h_query_scalars<F: PrimeField, D: EvaluationDomain<F>>(
        max_power: usize,
        t: F,
        _zt: F,
        delta_inverse: F,
    ) -> Result<Vec<F>, SynthesisError> {
        let n2 = 2 * (max_power + 1);
        let domain = D::new(n2).ok_or(SynthesisError::PolynomialDegreeTooLarge)?;
        let mut v = Vec::with_capacity(n2);
        let mut p = delta_inverse;
        for _ in 0..n2 - 1 {
            v.push(p);
            p *= t;
        }
        v.push(F::zero());
        domain.ifft_in_place(&mut v);
        Ok(v.into_iter().skip(1).step_by(2).collect())
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
