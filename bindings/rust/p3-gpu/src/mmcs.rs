//! `Mmcs` on the GPU: `MerkleTreeMmcs::commit` (`merkle-tree/src/mmcs/batch.rs:42-64`, `merkle_tree.rs:95-178`).
//! Openings and verification reuse the reference's own code on the returned `MerkleTree`.
use std::sync::Arc;

use p3_commit::Mmcs;
use p3_matrix::Matrix;
use p3_matrix::dense::RowMajorMatrix;
use p3_merkle_tree::{MerkleTree, MerkleTreeMmcs};
use p3_symmetric::MerkleCap;

use crate::ffi::*;
use crate::{GpuCtx, GpuField};

/// Which of the reference's hash configurations the GPU runs (`examples/src/types.rs:19-53`,
/// `keccak-air/examples/prove_baby_bear_sha256*.rs`); the discriminants are the ABI's `P3GPU_HASH_*`.
#[derive(Clone, Copy)]
pub enum GpuHash {
    /// `PaddingFreeSponge<Perm16,16,8,8>` + `TruncatedPermutation<Perm16,2,8,16>`
    Poseidon2W16 = P3GPU_HASH_POSEIDON2_W16 as isize,
    /// `PaddingFreeSponge<Perm24,24,16,8>` + `TruncatedPermutation<Perm16,2,8,16>`
    Poseidon2W24 = P3GPU_HASH_POSEIDON2_W24 as isize,
    /// `SerializingHasher<PaddingFreeSponge<KeccakF,25,17,4>>` + `CompressionFunctionFromHasher<_,2,4>`
    Keccak = P3GPU_HASH_KECCAK as isize,
    /// `SerializingHasher<Sha256>` + `CompressionFunctionFromHasher<Sha256,2,32>` (`[u8; 32]` digests)
    Sha256 = P3GPU_HASH_SHA256 as isize,
    /// `SerializingHasher<Sha256>` + `Sha256Compress` (`[u8; 32]` digests)
    Sha256Compress = P3GPU_HASH_SHA256_COMPRESS as isize,
}

/// Wraps the reference MMCS (`inner`, used for `open_batch` / `verify_batch` and for its hash parameters) and replaces `commit`.
#[derive(Clone)]
pub struct GpuMerkleMmcs<F, Inner> {
    pub(crate) ctx: Arc<GpuCtx>,
    pub(crate) hash: GpuHash,
    pub(crate) cap_height: usize,
    pub(crate) inner: Inner,
    _f: core::marker::PhantomData<F>,
}

impl<F: GpuField, Inner> GpuMerkleMmcs<F, Inner> {
    /// `rc16` / `rc24`: the Poseidon2 round constants Rust drew (`Poseidon2::new_from_rng_128`), as Montgomery words:
    /// (initial 4 x width, terminal 4 x width, internal R_P).
    pub fn new(ctx: Arc<GpuCtx>, hash: GpuHash, cap_height: usize, inner: Inner, rc16: Option<(&[u32], &[u32], &[u32])>,
               rc24: Option<(&[u32], &[u32], &[u32])>) -> Self {
        for (width, rc) in [(16, rc16), (24, rc24)] {
            if let Some((a, b, c)) = rc {
                check(unsafe { p3gpu_poseidon2_set_constants(ctx.raw(), F::GPU_ID, width, a.as_ptr(), b.as_ptr(), c.as_ptr(), c.len() as i32) });
            }
        }
        Self { ctx, hash, cap_height, inner, _f: core::marker::PhantomData }
    }
}

impl<F, P, PW, H, C, const DIGEST: usize> Mmcs<F> for GpuMerkleMmcs<F, MerkleTreeMmcs<P, PW, H, C, 2, DIGEST>>
where
    F: GpuField,
    MerkleTreeMmcs<P, PW, H, C, 2, DIGEST>: Mmcs<F, ProverData<RowMajorMatrix<F>> = MerkleTree<F, F, RowMajorMatrix<F>, 2, DIGEST>,
                                                   Commitment = MerkleCap<F, [F; DIGEST]>>,
{
    type ProverData<M> = <MerkleTreeMmcs<P, PW, H, C, 2, DIGEST> as Mmcs<F>>::ProverData<M>;
    type Commitment = <MerkleTreeMmcs<P, PW, H, C, 2, DIGEST> as Mmcs<F>>::Commitment;
    type Proof = <MerkleTreeMmcs<P, PW, H, C, 2, DIGEST> as Mmcs<F>>::Proof;
    type MultiProof = <MerkleTreeMmcs<P, PW, H, C, 2, DIGEST> as Mmcs<F>>::MultiProof;
    type Error = <MerkleTreeMmcs<P, PW, H, C, 2, DIGEST> as Mmcs<F>>::Error;

    fn commit<M: Matrix<F>>(&self, inputs: Vec<M>) -> (Self::Commitment, Self::ProverData<M>) {
        assert!(!inputs.is_empty(), "No matrices given?");
        // dense inputs are borrowed as they are (zero copy); other matrix types are materialised once
        let dense: Vec<RowMajorMatrix<F>> = inputs.iter().map(|m| m.to_row_major_matrix()).collect();
        let ptrs: Vec<*const u32> = dense.iter().map(|m| m.values.as_ptr().cast()).collect();
        let (hs, ws): (Vec<usize>, Vec<usize>) = dense.iter().map(|m| (m.height(), m.width())).unzip();
        let total = unsafe { p3gpu_merkle_total_digests(*hs.iter().max().unwrap()) };
        let mut flat = vec![[F::ZERO; DIGEST]; total];
        let (mut lens, mut n) = ([0usize; 65], 0usize);
        check(unsafe {
            p3gpu_merkle_commit(self.ctx.raw(), F::GPU_ID, self.hash as i32, ptrs.len(), ptrs.as_ptr(), hs.as_ptr(), ws.as_ptr(),
                                flat.as_mut_ptr().cast(), lens.as_mut_ptr(), &mut n)
        });
        let mut layers = Vec::with_capacity(n);
        let mut rest = flat.as_slice();
        for &len in &lens[..n] {
            let (layer, tail) = rest.split_at(len);
            layers.push(layer.to_vec());
            rest = tail;
        }
        // needs `MerkleTree::from_parts(leaves, digest_layers, arity_schedule)`: the struct's fields are pub(crate)
        // (merkle_tree.rs:33-69) — the one upstream change this shim asks for
        let tree = MerkleTree::from_parts(inputs, layers, vec![2; n - 1]);
        let cap = tree.cap(self.cap_height.min(n - 1));
        (cap, tree)
    }

    fn open_batch<M: Matrix<F>>(&self, index: usize, prover_data: &Self::ProverData<M>) -> p3_commit::BatchOpening<F, Self> {
        self.inner.open_batch(index, prover_data).map_mmcs()
    }
    fn get_matrices<'a, M: Matrix<F>>(&self, prover_data: &'a Self::ProverData<M>) -> Vec<&'a M> {
        self.inner.get_matrices(prover_data)
    }
    fn verify_batch(&self, commit: &Self::Commitment, dimensions: &[p3_matrix::Dimensions], index: usize,
                    batch_opening: p3_commit::BatchOpeningRef<'_, F, Self>) -> Result<(), Self::Error> {
        self.inner.verify_batch(commit, dimensions, index, batch_opening.map_mmcs())
    }
}
