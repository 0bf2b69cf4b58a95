//! Safe wrapper: a device-backed matrix with sprs's product call shapes.
//!
//! Orphan rules forbid re-implementing `Mul` for the foreign `CsMatBase`, so the
//! drop-in is a newtype owning the host `CsMatI` plus its device mirror (SURVEY 8b):
//!
//! ```ignore
//! let a = DeviceCsMat::new(a_host)?;        // uploads once (proper_indptr + as_ptr)
//! let y: Array1<f64> = &a * &x;             // csmat.rs:2119-2160 -> sprs_b200_mul_mat_vec
//! let c: Array2<f64> = &a * &b;             // csmat.rs:1989-2048 (k >= 8 -> rowmaj, C order)
//! let p: CsMatI<f64, I, Iptr> = &a * &b_sp; // csmat.rs:1866-1949 -> smmp::mul_csr_csr
//! let s: CsMatI<f64, I, Iptr> = &a + &b_sp; // binop.rs:20-112 (also `-`, `&a * 2.0`,
//!                                           // binop::mul_mat_same_storage)
//! ```
//! Contract violations panic with the reference's messages (Guidelines.rst:9-27);
//! device failures are `LinalgError::ThirdPartyError(code, msg)` (errors.rs:70).
use ndarray::{Array1, Array2, ArrayBase, ArrayView1, Data, Ix1, Ix2, ShapeBuilder};
use sprs::errors::LinalgError;
use sprs::{CsMatI, CsMatViewI, CsVecI, SpIndex};
use sprs_b200_sys as ffi;
use std::ffi::CStr;
use std::ops::Mul;
use std::os::raw::c_void;

thread_local! { static CTX: Ctx = Ctx::new(0).expect("no H100 device"); }

struct Ctx(*mut ffi::sprs_b200_ctx);
impl Ctx {
    fn new(device: i32) -> Result<Self, LinalgError> {
        let mut h = std::ptr::null_mut();
        let st = unsafe { ffi::sprs_b200_ctx_create(device, &mut h) };
        if st != ffi::SPRS_B200_OK { return Err(third_party(std::ptr::null(), st)); }
        Ok(Ctx(h))
    }
}
impl Drop for Ctx { fn drop(&mut self) { unsafe { ffi::sprs_b200_ctx_destroy(self.0); } } }

fn third_party(ctx: *const ffi::sprs_b200_ctx, code: i32) -> LinalgError {
    // errors.rs:70 wants a &'static str; leak the (rare) message like a panic payload
    let msg = unsafe { CStr::from_ptr(ffi::sprs_b200_last_error(ctx)) }.to_string_lossy().into_owned();
    LinalgError::ThirdPartyError(code as isize, Box::leak(msg.into_boxed_str()))
}
fn check(ctx: *const ffi::sprs_b200_ctx, st: i32) -> Result<(), LinalgError> {
    match st {
        ffi::SPRS_B200_OK => Ok(()),
        ffi::SPRS_B200_ERR_DIMENSION => panic!("Dimension mismatch"),
        ffi::SPRS_B200_ERR_STORAGE => panic!("Storage mismatch"),
        _ => Err(third_party(ctx, st)),
    }
}

/// Host `CsMatI` + device mirror; the mirror is released in `Drop` (UMFPACK pattern,
/// sprs_suitesparse_umfpack/src/lib.rs:33-46).
pub struct DeviceCsMat<I: SpIndex, Iptr: SpIndex = I> {
    host: CsMatI<f64, I, Iptr>,
    dev: *mut ffi::sprs_b200_csmat,
}

impl<I: SpIndex, Iptr: SpIndex> DeviceCsMat<I, Iptr> {
    pub fn new(host: CsMatI<f64, I, Iptr>) -> Result<Self, LinalgError> {
        assert!(matches!(std::mem::size_of::<I>(), 4 | 8) && matches!(std::mem::size_of::<Iptr>(), 4 | 8),
                "device mirrors take 4- or 8-byte index types; use to_other_types() first");
        let dev = upload(host.view())?;
        Ok(Self { host, dev })
    }
    pub fn host(&self) -> &CsMatI<f64, I, Iptr> { &self.host }
}
impl<I: SpIndex, Iptr: SpIndex> Drop for DeviceCsMat<I, Iptr> {
    fn drop(&mut self) { unsafe { ffi::sprs_b200_csmat_free(self.dev); } }
}

fn upload<I: SpIndex, Iptr: SpIndex>(m: CsMatViewI<f64, I, Iptr>) -> Result<*mut ffi::sprs_b200_csmat, LinalgError> {
    // like the reference's own FFI callers (sprs-benches/src/main.rs:55-58): proper
    // (zero-based) indptr and raw as_ptr(); the library rebases anyway.
    let indptr = m.proper_indptr();
    let mut out = std::ptr::null_mut();
    CTX.with(|c| check(c.0, unsafe {
        ffi::sprs_b200_csmat_upload(
            c.0, if m.is_csr() { ffi::SPRS_B200_CSR } else { ffi::SPRS_B200_CSC },
            m.rows() as u64, m.cols() as u64,
            indptr.as_ptr() as *const c_void, std::mem::size_of::<Iptr>() as i32,
            m.indices().as_ptr() as *const c_void, std::mem::size_of::<I>() as i32,
            m.data().as_ptr(), &mut out)
    }))?;
    Ok(out)
}

// `&A * &x`  (csmat.rs:2119-2160)
impl<'a, 'b, I: SpIndex, Iptr: SpIndex, DS: Data<Elem = f64>> Mul<&'b ArrayBase<DS, Ix1>> for &'a DeviceCsMat<I, Iptr> {
    type Output = Array1<f64>;
    fn mul(self, rhs: &'b ArrayBase<DS, Ix1>) -> Array1<f64> {
        assert_eq!(self.host.cols(), rhs.len(), "Dimension mismatch");
        let x = rhs.as_standard_layout();
        let mut y = Array1::<f64>::zeros(self.host.rows());
        CTX.with(|c| check(c.0, unsafe {
            ffi::sprs_b200_mul_mat_vec(c.0, self.dev, x.as_ptr(), x.len() as u64,
                                       y.as_mut_ptr(), y.len() as u64)
        })).expect("sprs_b200 device error");
        y
    }
}

// `&A * &v`, v sparse (vec.rs:1104-1131 -> prod::csr_mul_csvec, prod.rs:162-184): the per-row
// sorted-merge dot runs on the device (bit-identical); zeros are dropped here (prod.rs:178-180).
// A CSC lhs goes through the sparse-sparse product with `rhs.col_view()` like the reference.
impl<'a, 'b, I: SpIndex, Iptr: SpIndex> Mul<&'b CsVecI<f64, I>> for &'a DeviceCsMat<I, Iptr> {
    type Output = CsVecI<f64, I>;
    fn mul(self, rhs: &'b CsVecI<f64, I>) -> CsVecI<f64, I> {
        if rhs.dim() == 0 { return CsVecI::empty(0); }
        assert_eq!(self.host.cols(), rhs.dim(), "Dimension mismatch");
        assert!(self.host.is_csr(), "CSC x CsVec: use &a * &DeviceCsMat::new(rhs.col_view().to_owned())");
        let mut y = vec![0f64; self.host.rows()];
        CTX.with(|c| check(c.0, unsafe {
            ffi::sprs_b200_csr_mul_csvec(c.0, self.dev, rhs.dim() as u64, rhs.nnz() as u64,
                rhs.indices().as_ptr() as *const c_void, std::mem::size_of::<I>() as i32,
                rhs.data().as_ptr(), y.as_mut_ptr(), y.len() as u64)
        })).expect("sprs_b200 device error");
        let mut res = CsVecI::empty(self.host.rows());
        for (row, val) in y.into_iter().enumerate() {
            if val != 0.0 { res.append(row, val); }
        }
        res
    }
}

// `&A * &B`, dense B (csmat.rs:1989-2048): k >= 8 -> rowmaj kernel, C-order result
impl<'a, 'b, I: SpIndex, Iptr: SpIndex, DS: Data<Elem = f64>> Mul<&'b ArrayBase<DS, Ix2>> for &'a DeviceCsMat<I, Iptr> {
    type Output = Array2<f64>;
    fn mul(self, rhs: &'b ArrayBase<DS, Ix2>) -> Array2<f64> {
        let (rows, cols) = (self.host.rows(), rhs.shape()[1]);
        let (rs, cs) = (rhs.strides()[0] as i64, rhs.strides()[1] as i64);
        let wide = cols >= 8; // csmat.rs:2009
        let mut res = if wide { Array2::zeros((rows, cols)) } else { Array2::zeros((rows, cols).f()) };
        let (ors, ocs) = (res.strides()[0] as i64, res.strides()[1] as i64);
        let f = match (self.host.is_csr(), wide) {
            (true, true) => ffi::sprs_b200_csr_mulacc_dense_rowmaj,
            (true, false) => ffi::sprs_b200_csr_mulacc_dense_colmaj,
            (false, true) => ffi::sprs_b200_csc_mulacc_dense_rowmaj,
            (false, false) => ffi::sprs_b200_csc_mulacc_dense_colmaj,
        };
        CTX.with(|c| check(c.0, unsafe {
            f(c.0, self.dev, rhs.as_ptr(), rhs.shape()[0] as u64, cols as u64, rs, cs,
              res.as_mut_ptr(), rows as u64, cols as u64, ors, ocs)
        })).expect("sprs_b200 device error");
        res
    }
}

/// smmp::mul_csr_csr (smmp.rs:196-237): Rust allocates the output Vecs between the
/// symbolic and numeric calls, exactly where the reference does.
pub fn mul_csr_csr<I: SpIndex, Iptr: SpIndex>(lhs: &DeviceCsMat<I, Iptr>, rhs: &DeviceCsMat<I, Iptr>) -> CsMatI<f64, I, Iptr> {
    assert_eq!(lhs.host.cols(), rhs.host.rows());
    assert!(lhs.host.is_csr() && rhs.host.is_csr(), "Storage mismatch");
    CTX.with(|c| {
        let (mut plan, mut nnz_c) = (std::ptr::null_mut(), 0u64);
        check(c.0, unsafe { ffi::sprs_b200_spgemm_symbolic(c.0, lhs.dev, rhs.dev, &mut plan, &mut nnz_c) })
            .expect("sprs_b200 device error");
        let mut indptr = vec![Iptr::zero(); lhs.host.rows() + 1];
        let mut indices = vec![I::zero(); nnz_c as usize];
        let mut data = vec![0f64; nnz_c as usize];
        let st = unsafe {
            ffi::sprs_b200_spgemm_numeric(c.0, plan, indptr.as_mut_ptr() as *mut c_void,
                std::mem::size_of::<Iptr>() as i32, indices.as_mut_ptr() as *mut c_void,
                std::mem::size_of::<I>() as i32, data.as_mut_ptr())
        };
        unsafe { ffi::sprs_b200_spgemm_free(plan); }
        check(c.0, st).expect("sprs_b200 device error");
        // invariants hold by construction (sorted unique in-range columns): smmp.rs:406-415
        CsMatI::new_trusted(sprs::CompressedStorage::CSR, (lhs.host.rows(), rhs.host.cols()), indptr, indices, data)
    })
}

// `&A * &B`, both sparse (csmat.rs:1866-1949) for the (CSR, CSR) case; the mixed-storage
// arms convert with to_other_storage() exactly as csmat_mul_csmat does.
impl<'a, 'b, I: SpIndex, Iptr: SpIndex> Mul<&'b DeviceCsMat<I, Iptr>> for &'a DeviceCsMat<I, Iptr> {
    type Output = CsMatI<f64, I, Iptr>;
    fn mul(self, rhs: &'b DeviceCsMat<I, Iptr>) -> Self::Output { mul_csr_csr(self, rhs) }
}

// ---- binop.rs:20-163: `&A + &B`, `&A - &B`, `&A * s` and binop::mul_mat_same_storage.  The
// device result (lhs storage, entries whose result is 0.0 dropped; map keeps every entry) is
// downloaded into Vecs the caller side allocates, like mul_csr_csr.
fn download_result<I: SpIndex, Iptr: SpIndex>(c: *mut ffi::sprs_b200_ctx, m: *mut ffi::sprs_b200_csmat,
                                              like: &CsMatI<f64, I, Iptr>) -> CsMatI<f64, I, Iptr> {
    let nnz = unsafe { ffi::sprs_b200_csmat_nnz(m) } as usize;
    let mut indptr = vec![Iptr::zero(); like.outer_dims() + 1];
    let mut indices = vec![I::zero(); nnz];
    let mut data = vec![0f64; nnz];
    let st = unsafe {
        ffi::sprs_b200_csmat_download(c, m, indptr.as_mut_ptr() as *mut c_void,
            std::mem::size_of::<Iptr>() as i32, indices.as_mut_ptr() as *mut c_void,
            std::mem::size_of::<I>() as i32, data.as_mut_ptr())
    };
    unsafe { ffi::sprs_b200_csmat_free(m); }
    check(c, st).expect("sprs_b200 device error");
    // sorted unique in-range indices by construction (binop.rs:210-217 new_trusted)
    CsMatI::new_trusted(like.storage(), (like.rows(), like.cols()), indptr, indices, data)
}

fn csmat_binop<I: SpIndex, Iptr: SpIndex>(lhs: &DeviceCsMat<I, Iptr>, rhs: &DeviceCsMat<I, Iptr>, op: i32) -> CsMatI<f64, I, Iptr> {
    // binop.rs:195-199: shapes first, then storage; Add / Sub convert rhs (binop.rs:20-112)
    assert!(lhs.host.rows() == rhs.host.rows() && lhs.host.cols() == rhs.host.cols(), "Dimension mismatch");
    CTX.with(|c| {
        let mut conv = std::ptr::null_mut();
        let rdev = if lhs.host.storage() == rhs.host.storage() { rhs.dev } else {
            assert!(op != ffi::SPRS_B200_BINOP_MUL, "Storage mismatch");
            check(c.0, unsafe { ffi::sprs_b200_csmat_to_other_storage(c.0, rhs.dev, &mut conv) })
                .expect("sprs_b200 device error");
            conv
        };
        let mut out = std::ptr::null_mut();
        let st = unsafe { ffi::sprs_b200_csmat_binop(c.0, lhs.dev, rdev, op, &mut out) };
        if !conv.is_null() { unsafe { ffi::sprs_b200_csmat_free(conv); } }
        check(c.0, st).expect("sprs_b200 device error");
        download_result(c.0, out, &lhs.host)
    })
}

impl<'a, 'b, I: SpIndex, Iptr: SpIndex> std::ops::Add<&'b DeviceCsMat<I, Iptr>> for &'a DeviceCsMat<I, Iptr> {
    type Output = CsMatI<f64, I, Iptr>;
    fn add(self, rhs: &'b DeviceCsMat<I, Iptr>) -> Self::Output { csmat_binop(self, rhs, ffi::SPRS_B200_BINOP_ADD) }
}
impl<'a, 'b, I: SpIndex, Iptr: SpIndex> std::ops::Sub<&'b DeviceCsMat<I, Iptr>> for &'a DeviceCsMat<I, Iptr> {
    type Output = CsMatI<f64, I, Iptr>;
    fn sub(self, rhs: &'b DeviceCsMat<I, Iptr>) -> Self::Output { csmat_binop(self, rhs, ffi::SPRS_B200_BINOP_SUB) }
}
// `&A * s` (binop.rs:132-163 -> CsMatBase::map): same structure, every value times s
impl<'a, I: SpIndex, Iptr: SpIndex> Mul<f64> for &'a DeviceCsMat<I, Iptr> {
    type Output = CsMatI<f64, I, Iptr>;
    fn mul(self, s: f64) -> Self::Output {
        CTX.with(|c| {
            let mut out = std::ptr::null_mut();
            check(c.0, unsafe { ffi::sprs_b200_csmat_scale(c.0, self.dev, s, &mut out) })
                .expect("sprs_b200 device error");
            download_result(c.0, out, &self.host)
        })
    }
}

pub mod binop {
    use super::*;
    /// binop::mul_mat_same_storage (binop.rs:115-130): element-wise product; mixed storage
    /// panics "Storage mismatch" (no conversion).
    pub fn mul_mat_same_storage<I: SpIndex, Iptr: SpIndex>(lhs: &DeviceCsMat<I, Iptr>, rhs: &DeviceCsMat<I, Iptr>) -> CsMatI<f64, I, Iptr> {
        super::csmat_binop(lhs, rhs, ffi::SPRS_B200_BINOP_MUL)
    }
}

/// The dense boundary on the device (the dense section of csrc/transpose.cu): to_dense.rs, CsMat::csr_from_dense /
/// csc_from_dense (csmat.rs:502-549) and the sparse (+) dense half of binop.rs, bit-identical
/// to the reference.  Views of any strides are passed as (pointer, shape, element strides);
/// ndarray gives a view with a zero-length axis all-zero strides, and so does this crate.
pub mod dense {
    use super::*;
    use ndarray::{Array2, ArrayBase, ArrayViewMut2, Data, Ix2, ShapeBuilder};

    fn strides<S: ndarray::RawData>(a: &ArrayBase<S, Ix2>) -> (i64, i64) {
        if a.is_empty() { (0, 0) } else { (a.strides()[0] as i64, a.strides()[1] as i64) }
    }
    fn c_like<S: ndarray::RawData>(a: &ArrayBase<S, Ix2>) -> bool {
        let (rs, cs) = strides(a);
        !(cs > rs)  // utils::fastest_axis (sparse.rs:400-406)
    }

    /// CsMat::to_dense (csmat.rs:1127-1134): C order, stored values as bits, +0.0 elsewhere.
    pub fn to_dense<I: SpIndex, Iptr: SpIndex>(m: &DeviceCsMat<I, Iptr>) -> Array2<f64> {
        let (r, c) = (m.host.rows(), m.host.cols());
        let mut out = Array2::<f64>::zeros((r, c));
        if r > 0 && c > 0 {
            CTX.with(|x| check(x.0, unsafe {
                ffi::sprs_b200_csmat_to_dense(x.0, m.dev, out.as_mut_ptr(), c as u64) }))
                .expect("sprs_b200 device error");
        }
        out
    }

    /// assign_to_dense (to_dense.rs:12-30): every stored value into `array`, the rest untouched.
    pub fn assign_to_dense<I: SpIndex, Iptr: SpIndex>(mut array: ArrayViewMut2<f64>, m: &DeviceCsMat<I, Iptr>) {
        assert_eq!(m.host.cols(), array.shape()[1], "Dimension mismatch");
        assert_eq!(m.host.rows(), array.shape()[0], "Dimension mismatch");
        let (rs, cs) = strides(&array);
        let (r, c) = (array.shape()[0] as u64, array.shape()[1] as u64);
        CTX.with(|x| check(x.0, unsafe {
            ffi::sprs_b200_assign_to_dense(x.0, m.dev, array.as_mut_ptr(), r, c, rs, cs) }))
            .expect("sprs_b200 device error");
    }

    fn from_dense<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(m: &ArrayBase<S, Ix2>, epsilon: f64, csr: bool) -> CsMatI<f64, I, Iptr> {
        let (rs, cs) = strides(m);
        let (r, c) = (m.shape()[0], m.shape()[1]);
        let st = if csr { ffi::SPRS_B200_CSR } else { ffi::SPRS_B200_CSC };
        CTX.with(|x| {
            let mut out = std::ptr::null_mut();
            check(x.0, unsafe { ffi::sprs_b200_csmat_from_dense(x.0, st, r as u64, c as u64, m.as_ptr(),
                                                                rs, cs, epsilon, &mut out) })
                .expect("sprs_b200 device error");
            let like: CsMatI<f64, I, Iptr> = if csr { CsMatI::zero((r, c)) } else { CsMatI::zero((r, c)).to_csc() };
            download_result(x.0, out, &like)
        })
    }
    /// CsMat::csr_from_dense (csmat.rs:502-539): |x| > epsilon kept (epsilon clamped to +0.0
    /// unless > 0), values as bits, columns ascending in each row.
    pub fn csr_from_dense<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(m: &ArrayBase<S, Ix2>, epsilon: f64) -> CsMatI<f64, I, Iptr> {
        from_dense(m, epsilon, true)
    }
    /// CsMat::csc_from_dense (csmat.rs:544-549).
    pub fn csc_from_dense<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(m: &ArrayBase<S, Ix2>, epsilon: f64) -> CsMatI<f64, I, Iptr> {
        from_dense(m, epsilon, false)
    }

    fn binop_dense<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(lhs: *const ffi::sprs_b200_csmat, op: i32, alpha: f64,
                                                                   beta: f64, rhs: &ArrayBase<S, Ix2>) -> Array2<f64> {
        let shape = (rhs.shape()[0], rhs.shape()[1]);
        let mut out = if c_like(rhs) { Array2::zeros(shape) } else { Array2::zeros(shape.f()) };
        let (rrs, rcs) = strides(rhs);
        let (ors, ocs) = strides(&out);
        CTX.with(|x| check(x.0, unsafe {
            ffi::sprs_b200_csmat_binop_dense(x.0, lhs, op, alpha, beta, rhs.as_ptr(), shape.0 as u64,
                                             shape.1 as u64, rrs, rcs, out.as_mut_ptr(), shape.0 as u64,
                                             shape.1 as u64, ors, ocs) }))
            .expect("sprs_b200 device error");
        out
    }
    /// binop::add_dense_mat_same_ordering (binop.rs:279-323): (alpha*x) + (beta*y).
    pub fn add_dense_mat_same_ordering<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(
        lhs: &DeviceCsMat<I, Iptr>, rhs: &ArrayBase<S, Ix2>, alpha: f64, beta: f64) -> Array2<f64> {
        binop_dense::<S, I, Iptr>(lhs.dev, ffi::SPRS_B200_BINOP_ADD, alpha, beta, rhs)
    }
    /// binop::mul_dense_mat_same_ordering (binop.rs:331-371): (alpha*x)*y.
    pub fn mul_dense_mat_same_ordering<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(
        lhs: &DeviceCsMat<I, Iptr>, rhs: &ArrayBase<S, Ix2>, alpha: f64) -> Array2<f64> {
        binop_dense::<S, I, Iptr>(lhs.dev, ffi::SPRS_B200_BINOP_MUL, alpha, 0.0, rhs)
    }
    /// `&A + &D` (csmat.rs:1951-1987): A converted first when its storage does not match D's
    /// fastest axis; the result has D's layout.
    pub fn add_dense<S: Data<Elem = f64>, I: SpIndex, Iptr: SpIndex>(a: &DeviceCsMat<I, Iptr>, d: &ArrayBase<S, Ix2>) -> Array2<f64> {
        if a.host.is_csr() == c_like(d) { return add_dense_mat_same_ordering(a, d, 1.0, 1.0); }
        CTX.with(|x| {
            let mut conv = std::ptr::null_mut();
            check(x.0, unsafe { ffi::sprs_b200_csmat_to_other_storage(x.0, a.dev, &mut conv) })
                .expect("sprs_b200 device error");
            let out = binop_dense::<S, I, Iptr>(conv, ffi::SPRS_B200_BINOP_ADD, 1.0, 1.0, d);
            unsafe { ffi::sprs_b200_csmat_free(conv); }
            out
        })
    }
}

/// sprs::bmat / vstack / hstack (construct.rs) and sprs::kronecker_product (kronecker.rs) on the
/// device, bit-identical to the reference (csrc/construct.cu).  The asserts run here in the
/// reference's order; a result dimension >= 2^32 is a device error (u32 mirrors) even where
/// usize would allow it.
pub mod construct {
    use super::*;
    use sprs::CompressedStorage::{CSC, CSR};

    fn download_as<I: SpIndex, Iptr: SpIndex>(c: *mut ffi::sprs_b200_ctx, m: *mut ffi::sprs_b200_csmat,
                                              storage: sprs::CompressedStorage,
                                              shape: (usize, usize)) -> CsMatI<f64, I, Iptr> {
        let outer = if storage == CSR { shape.0 } else { shape.1 };
        let nnz = unsafe { ffi::sprs_b200_csmat_nnz(m) } as usize;
        let mut indptr = vec![Iptr::zero(); outer + 1];
        let mut indices = vec![I::zero(); nnz];
        let mut data = vec![0f64; nnz];
        let st = unsafe {
            ffi::sprs_b200_csmat_download(c, m, indptr.as_mut_ptr() as *mut c_void,
                std::mem::size_of::<Iptr>() as i32, indices.as_mut_ptr() as *mut c_void,
                std::mem::size_of::<I>() as i32, data.as_mut_ptr())
        };
        unsafe { ffi::sprs_b200_csmat_free(m); }
        check(c, st).expect("sprs_b200 device error");
        // sorted unique in-range indices by construction
        CsMatI::new_trusted(storage, shape, indptr, indices, data)
    }

    /// bmat (construct.rs): always CSR; `None` is zero((max rows of its block row, max cols of
    /// its block column)).
    pub fn bmat<I: SpIndex, Iptr: SpIndex>(blocks: &[Vec<Option<&DeviceCsMat<I, Iptr>>>]) -> CsMatI<f64, I, Iptr> {
        assert_ne!(blocks.len(), 0, "Empty stacking list");
        let nbc = blocks[0].len();
        assert_ne!(nbc, 0, "Empty stacking list");
        assert!(blocks.iter().all(|r| r.len() == nbc), "Dimension mismatch");
        assert!(!blocks.iter().any(|r| r.iter().all(Option::is_none)), "Empty bmat row");
        assert!(!(0..nbc).any(|j| blocks.iter().all(|r| r[j].is_none())), "Empty bmat col");
        let widths: Vec<usize> = (0..nbc)
            .map(|j| blocks.iter().filter_map(|r| r[j].map(|m| m.host.cols())).max().unwrap_or(0))
            .collect();
        let rows: usize = blocks.iter()
            .map(|r| r.iter().filter_map(|m| m.map(|m| m.host.rows())).max().unwrap_or(0)).sum();
        let cols: usize = blocks[0].iter().zip(&widths).map(|(m, w)| m.map_or(*w, |m| m.host.cols())).sum();
        let grid: Vec<*const ffi::sprs_b200_csmat> = blocks.iter()
            .flat_map(|r| r.iter().map(|m| m.map_or(std::ptr::null(), |m| m.dev as *const _)))
            .collect();
        CTX.with(|c| {
            let mut out = std::ptr::null_mut();
            check(c.0, unsafe { ffi::sprs_b200_csmat_bmat(c.0, blocks.len() as u64, nbc as u64, grid.as_ptr(), &mut out) })
                .expect("sprs_b200 device error");
            download_as(c.0, out, CSR, (rows, cols))
        })
    }

    /// vstack (construct.rs): the CSR forms stacked vertically; always CSR.
    pub fn vstack<I: SpIndex, Iptr: SpIndex>(mats: &[&DeviceCsMat<I, Iptr>]) -> CsMatI<f64, I, Iptr> {
        assert!(!mats.is_empty(), "Empty stacking list");
        let col: Vec<Vec<Option<&DeviceCsMat<I, Iptr>>>> = mats.iter().map(|m| vec![Some(*m)]).collect();
        bmat(&col)
    }

    /// hstack (construct.rs): the CSC forms stacked horizontally; always CSC.  On the device it
    /// is the vstack of the blocks' transpose views, read back as the CSC it is.
    pub fn hstack<I: SpIndex, Iptr: SpIndex>(mats: &[&DeviceCsMat<I, Iptr>]) -> CsMatI<f64, I, Iptr> {
        assert!(!mats.is_empty(), "Empty stacking list");
        CTX.with(|c| {
            let mut views: Vec<*const ffi::sprs_b200_csmat> = Vec::with_capacity(mats.len());
            let mut st = ffi::SPRS_B200_OK;
            for m in mats {
                let mut v = std::ptr::null_mut();
                st = unsafe { ffi::sprs_b200_csmat_transpose_view(c.0, m.dev, &mut v) };
                if st != ffi::SPRS_B200_OK { break; }
                views.push(v);
            }
            let mut out = std::ptr::null_mut();
            if st == ffi::SPRS_B200_OK {
                st = unsafe { ffi::sprs_b200_csmat_bmat(c.0, views.len() as u64, 1, views.as_ptr(), &mut out) };
            }
            for v in views { unsafe { ffi::sprs_b200_csmat_free(v as *mut _); } }
            check(c.0, st).expect("sprs_b200 device error");
            let cols = mats.iter().map(|m| m.host.cols()).sum();
            download_as(c.0, out, CSC, (mats[0].host.rows(), cols))
        })
    }

    /// kronecker_product (kronecker.rs): in a's storage, b converted when the storages differ;
    /// a produced index that does not fit I panics like the reference's `unwrap()`.
    pub fn kronecker_product<I: SpIndex, Iptr: SpIndex>(a: &DeviceCsMat<I, Iptr>, b: &DeviceCsMat<I, Iptr>) -> CsMatI<f64, I, Iptr> {
        let (ha, hb) = (&a.host, &b.host);
        if ha.nnz() > 0 && hb.nnz() > 0 {
            let max_a = ha.indices().iter().map(|i| i.index()).max().unwrap_or(0);
            let (inner_b, max_b) = if hb.storage() == ha.storage() {
                (hb.inner_dims(), hb.indices().iter().map(|i| i.index()).max().unwrap_or(0))
            } else {
                let last = hb.indptr().to_proper().windows(2).rposition(|w| w[1] > w[0]).unwrap_or(0);
                (hb.outer_dims(), last)
            };
            let top = (max_a as u128) * (inner_b as u128) + max_b as u128;
            assert!(top <= I::max_value().index() as u128, "called `Option::unwrap()` on a `None` value");
        }
        CTX.with(|c| {
            let mut out = std::ptr::null_mut();
            check(c.0, unsafe { ffi::sprs_b200_csmat_kron(c.0, a.dev, b.dev, &mut out) })
                .expect("sprs_b200 device error");
            download_as(c.0, out, ha.storage(), (ha.rows() * hb.rows(), ha.cols() * hb.cols()))
        })
    }
}

/// sprs::linalg::bicgstab::BiCGSTAB<f64> (linalg/bicgstab.rs:95-300) with x, r, rhat, p
/// resident on the device between iterations.  Same constructor, `solve`, `step`,
/// restarts and accessors; vectors cross the API as dense `Array1<f64>`.
pub mod bicgstab {
    use super::*;
    pub struct BiCGSTAB<'a, I: SpIndex, Iptr: SpIndex> { a: &'a DeviceCsMat<I, Iptr>, h: *mut ffi::sprs_b200_bicgstab }
    impl<'a, I: SpIndex, Iptr: SpIndex> Drop for BiCGSTAB<'a, I, Iptr> {
        fn drop(&mut self) { unsafe { ffi::sprs_b200_bicgstab_free(self.h); } }
    }
    impl<'a, I: SpIndex, Iptr: SpIndex> BiCGSTAB<'a, I, Iptr> {
        /// bicgstab.rs:120-146
        pub fn new(a: &'a DeviceCsMat<I, Iptr>, x0: ArrayView1<f64>, b: ArrayView1<f64>) -> Self {
            assert_eq!(a.host.cols(), x0.len(), "Dimension mismatch");
            assert_eq!(a.host.rows(), b.len(), "Dimension mismatch");
            let (x0, b) = (x0.to_owned(), b.to_owned()); // contiguous
            let mut h = std::ptr::null_mut();
            CTX.with(|c| check(c.0, unsafe {
                ffi::sprs_b200_bicgstab_new(c.0, a.dev, x0.as_ptr(), b.as_ptr(), b.len() as u64, &mut h)
            })).expect("sprs_b200 device error");
            Self { a, h }
        }
        /// bicgstab.rs:151-175
        pub fn solve(a: &'a DeviceCsMat<I, Iptr>, x0: ArrayView1<f64>, b: ArrayView1<f64>, tol: f64,
                     max_iter: usize) -> Result<Box<Self>, Box<Self>> {
            let solver = Self::new(a, x0, b);
            let mut converged = 0;
            CTX.with(|c| check(c.0, unsafe {
                ffi::sprs_b200_bicgstab_solve(solver.h, tol, max_iter as u64, &mut converged)
            })).expect("sprs_b200 device error");
            if converged != 0 { Ok(Box::new(solver)) } else { Err(Box::new(solver)) }
        }
        pub fn step(&mut self) -> f64 {
            let mut err = 0.0;
            CTX.with(|c| check(c.0, unsafe { ffi::sprs_b200_bicgstab_step(self.h, &mut err) }))
                .expect("sprs_b200 device error");
            err
        }
        pub fn soft_restart(&mut self) { unsafe { ffi::sprs_b200_bicgstab_soft_restart(self.h); } }
        pub fn hard_restart(&mut self) { unsafe { ffi::sprs_b200_bicgstab_hard_restart(self.h); } }
        pub fn with_restart_threshold(self, thresh: f64) -> Self {
            unsafe { ffi::sprs_b200_bicgstab_set_restart_threshold(self.h, thresh); }
            self
        }
        fn stats(&self) -> ([u64; 3], [f64; 3]) {
            let (mut c, mut s) = ([0u64; 3], [0f64; 3]);
            unsafe { ffi::sprs_b200_bicgstab_stats(self.h, c.as_mut_ptr(), s.as_mut_ptr()); }
            (c, s)
        }
        pub fn iteration_count(&self) -> usize { self.stats().0[0] as usize }
        pub fn soft_restart_count(&self) -> usize { self.stats().0[1] as usize }
        pub fn hard_restart_count(&self) -> usize { self.stats().0[2] as usize }
        pub fn err(&self) -> f64 { self.stats().1[0] }
        pub fn rho(&self) -> f64 { self.stats().1[1] }
        pub fn soft_restart_threshold(&self) -> f64 { self.stats().1[2] }
        pub fn a(&self) -> &DeviceCsMat<I, Iptr> { self.a }
        fn vec(&self, which: i32) -> Array1<f64> {
            let mut out = Array1::zeros(self.a.host.rows());
            unsafe { ffi::sprs_b200_bicgstab_get(self.h, which, out.as_mut_ptr(), out.len() as u64); }
            out
        }
        pub fn x(&self) -> Array1<f64> { self.vec(ffi::SPRS_B200_BICGSTAB_X) }
        pub fn b(&self) -> Array1<f64> { self.vec(ffi::SPRS_B200_BICGSTAB_B) }
        pub fn r(&self) -> Array1<f64> { self.vec(ffi::SPRS_B200_BICGSTAB_R) }
        pub fn rhat(&self) -> Array1<f64> { self.vec(ffi::SPRS_B200_BICGSTAB_RHAT) }
        pub fn p(&self) -> Array1<f64> { self.vec(ffi::SPRS_B200_BICGSTAB_P) }
    }
}

/// sprs::linalg::trisolve (linalg/trisolve.rs:30-262) on the device: `rhs` solved in place,
/// bit-identical to the reference.  The reference's asserts panic with its messages in its
/// order (square, `rhs.dim()`, storage); a singular matrix is
/// `Err(LinalgError::SingularMatrix(SingularMatrixInfo { index, reason }))` with `rhs` left as
/// the reference leaves it.
pub mod linalg {
    pub mod trisolve {
        use super::super::*;
        use sprs::errors::SingularMatrixInfo;

        fn solve<I: SpIndex, Iptr: SpIndex>(mat: &DeviceCsMat<I, Iptr>, rhs: &mut [f64], tri: i32,
                                            csr: bool) -> Result<(), LinalgError> {
            assert_eq!(mat.host.cols(), mat.host.rows(), "Non square matrix passed to solver");
            assert_eq!(mat.host.cols(), rhs.len(), "Dimension mismatch");
            assert!(mat.host.is_csr() == csr, "Storage mismatch");
            CTX.with(|c| {
                let mut plan = std::ptr::null_mut();
                check(c.0, unsafe { ffi::sprs_b200_trisolve_plan(c.0, mat.dev, tri, &mut plan) })?;
                let st = unsafe { ffi::sprs_b200_trisolve_solve(plan, rhs.as_mut_ptr(), rhs.len() as u64) };
                let (mut index, mut reason) = (0u64, 0i32);
                let singular = unsafe { ffi::sprs_b200_trisolve_singular(plan, &mut index, &mut reason) } != 0;
                unsafe { ffi::sprs_b200_trisolve_free(plan); }
                if st == ffi::SPRS_B200_ERR_SINGULAR && singular {
                    let reason = match reason {
                        ffi::SPRS_B200_SINGULAR_IS_ZERO => "diagonal element is 0",
                        ffi::SPRS_B200_SINGULAR_NUMERIC => "diagonal element is a numeric 0",
                        _ => "diagonal element is a structural 0",
                    };
                    return Err(LinalgError::SingularMatrix(SingularMatrixInfo { index: index as usize, reason }));
                }
                check(c.0, st)
            })
        }
        /// trisolve.rs:30-73
        pub fn lsolve_csr_dense_rhs<I: SpIndex, Iptr: SpIndex>(lower_tri_mat: &DeviceCsMat<I, Iptr>, rhs: &mut [f64]) -> Result<(), LinalgError> {
            solve(lower_tri_mat, rhs, ffi::SPRS_B200_TRI_LOWER, true)
        }
        /// trisolve.rs:219-262
        pub fn usolve_csr_dense_rhs<I: SpIndex, Iptr: SpIndex>(upper_tri_mat: &DeviceCsMat<I, Iptr>, rhs: &mut [f64]) -> Result<(), LinalgError> {
            solve(upper_tri_mat, rhs, ffi::SPRS_B200_TRI_UPPER, true)
        }
        /// trisolve.rs:85-149
        pub fn lsolve_csc_dense_rhs<I: SpIndex, Iptr: SpIndex>(lower_tri_mat: &DeviceCsMat<I, Iptr>, rhs: &mut [f64]) -> Result<(), LinalgError> {
            solve(lower_tri_mat, rhs, ffi::SPRS_B200_TRI_LOWER, false)
        }
        /// trisolve.rs:161-210
        pub fn usolve_csc_dense_rhs<I: SpIndex, Iptr: SpIndex>(upper_tri_mat: &DeviceCsMat<I, Iptr>, rhs: &mut [f64]) -> Result<(), LinalgError> {
            solve(upper_tri_mat, rhs, ffi::SPRS_B200_TRI_UPPER, false)
        }
    }
}

/// The sprs-ldl crate (sprs-ldl/src/lib.rs) on the device: `LdlSymbolic` / `LdlNumeric` with the
/// reference's names, bit-identical L, D, x and singular index.  The permutation is the one
/// given (`new_perm`) or the identity (`new`); no fill-reducing ordering is computed.  Panics
/// follow the reference's order: square, symmetry (`CheckSymmetry`), permutation.  After an
/// `update` that returns `Err(SingularMatrix)`, `l`, `d` and `solve` panic until an `update`
/// succeeds; an `update` with another pattern panics before any work is done.
pub mod ldl {
    use super::*;
    use sprs::errors::SingularMatrixInfo;
    use sprs::SymmetryCheck;
    use std::rc::Rc;

    const NUMERIC_ZERO: &str = "diagonal element is a numeric 0";

    struct Handle(*mut ffi::sprs_b200_ldl);
    impl Drop for Handle { fn drop(&mut self) { unsafe { ffi::sprs_b200_ldl_free(self.0); } } }

    fn status(ctx: *const ffi::sprs_b200_ctx, st: i32, index: u64) -> Result<(), LinalgError> {
        match st {
            ffi::SPRS_B200_ERR_NOT_SYMMETRIC => panic!("Matrix is not symmetric"),
            ffi::SPRS_B200_ERR_SINGULAR => Err(LinalgError::SingularMatrix(SingularMatrixInfo {
                index: index as usize, reason: NUMERIC_ZERO })),
            ffi::SPRS_B200_ERR_STRUCTURE => panic!("{}", third_party(ctx, st)),
            _ => check(ctx, st),
        }
    }

    /// `sprs::is_symmetric` on the device.
    pub fn is_symmetric<I: SpIndex, Iptr: SpIndex>(mat: &DeviceCsMat<I, Iptr>) -> bool {
        CTX.with(|c| {
            let mut out = 0;
            check(c.0, unsafe { ffi::sprs_b200_is_symmetric(c.0, mat.dev, &mut out) }).unwrap();
            out != 0
        })
    }

    /// `sprs::linalg::diag_solve`: x_i /= diag_i on the device.
    pub fn diag_solve(diag: &[f64], x: &mut [f64]) {
        assert_eq!(diag.len(), x.len());
        CTX.with(|c| check(c.0, unsafe {
            ffi::sprs_b200_diag_solve(c.0, diag.as_ptr(), x.as_mut_ptr(), x.len() as u64) }).unwrap());
    }

    pub struct LdlSymbolic { h: Rc<Handle>, n: usize }
    impl LdlSymbolic {
        pub fn new<I: SpIndex, Iptr: SpIndex>(mat: &DeviceCsMat<I, Iptr>) -> Self {
            assert_eq!(mat.host.rows(), mat.host.cols());
            Self::new_perm(mat, None, SymmetryCheck::CheckSymmetry)
        }
        /// `perm[k]` is the outer vector of `mat` that is row k of P A P^T; `None`: identity.
        pub fn new_perm<I: SpIndex, Iptr: SpIndex>(mat: &DeviceCsMat<I, Iptr>, perm: Option<&[usize]>,
                                                  check_symmetry: SymmetryCheck) -> Self {
            let n = mat.host.rows();
            assert!(mat.host.cols() == n, "matrix should be square");
            let p: Option<Vec<u32>> = perm.map(|p| p.iter().map(|&v| v.min(u32::MAX as usize) as u32).collect());
            if let Some(p) = &p {
                if p.len() != n {
                    if check_symmetry == SymmetryCheck::CheckSymmetry && !is_symmetric(mat) {
                        panic!("Matrix is not symmetric");
                    }
                    panic!("assertion failed: perm_is_valid(&perm)");
                }
            }
            let check = (check_symmetry == SymmetryCheck::CheckSymmetry) as i32;
            CTX.with(|c| {
                let mut h = std::ptr::null_mut();
                let pp = p.as_ref().map_or(std::ptr::null(), |p| p.as_ptr());
                let st = unsafe { ffi::sprs_b200_ldl_symbolic(c.0, mat.dev, pp, check, &mut h) };
                if st == ffi::SPRS_B200_ERR_ARGUMENT { panic!("assertion failed: perm_is_valid(&perm)"); }
                if st == ffi::SPRS_B200_ERR_DIMENSION { panic!("matrix should be square"); }
                status(c.0, st, 0).unwrap();
                Self { h: Rc::new(Handle(h)), n }
            })
        }
        pub fn problem_size(&self) -> usize { self.n }
        pub fn nnz(&self) -> usize { unsafe { ffi::sprs_b200_ldl_nnz(self.h.0) as usize } }
        pub fn factor<I: SpIndex, Iptr: SpIndex>(self, mat: &DeviceCsMat<I, Iptr>) -> Result<LdlNumeric, LinalgError> {
            assert!(self.n > 1);  // DStack::with_capacity(n)
            CTX.with(|c| {
                let mut h = std::ptr::null_mut();
                let st = unsafe { ffi::sprs_b200_ldl_factor(self.h.0, mat.dev, &mut h) };
                let num = if h.is_null() { None } else { Some(Handle(h)) };
                let mut index = 0u64;
                if let Some(n) = &num { unsafe { ffi::sprs_b200_ldl_singular(n.0, &mut index); } }
                status(c.0, st, index)?;
                Ok(LdlNumeric { h: num.unwrap(), sym: self })
            })
        }
    }

    pub struct LdlNumeric { h: Handle, sym: LdlSymbolic }  // `h` drops before `sym`
    impl LdlNumeric {
        pub fn new<I: SpIndex, Iptr: SpIndex>(mat: &DeviceCsMat<I, Iptr>) -> Result<Self, LinalgError> {
            LdlSymbolic::new(mat).factor(mat)
        }
        pub fn new_perm<I: SpIndex, Iptr: SpIndex>(mat: &DeviceCsMat<I, Iptr>, perm: &[usize],
                                                  check_symmetry: SymmetryCheck) -> Result<Self, LinalgError> {
            LdlSymbolic::new_perm(mat, Some(perm), check_symmetry).factor(mat)
        }
        pub fn update<I: SpIndex, Iptr: SpIndex>(&mut self, mat: &DeviceCsMat<I, Iptr>) -> Result<(), LinalgError> {
            CTX.with(|c| {
                let st = unsafe { ffi::sprs_b200_ldl_update(self.h.0, mat.dev) };
                let mut index = 0u64;
                unsafe { ffi::sprs_b200_ldl_singular(self.h.0, &mut index); }
                status(c.0, st, index)
            })
        }
        fn valid(&self) {
            let mut index = 0u64;
            if unsafe { ffi::sprs_b200_ldl_singular(self.h.0, &mut index) } != 0 {
                panic!("Singular matrix at index {} ({})", index, NUMERIC_ZERO);
            }
        }
        pub fn solve(&self, rhs: &[f64]) -> Vec<f64> {
            assert_eq!(self.sym.n, rhs.len());
            self.valid();
            let mut x = vec![0.0; rhs.len()];
            CTX.with(|c| check(c.0, unsafe {
                ffi::sprs_b200_ldl_solve(self.h.0, rhs.as_ptr(), x.as_mut_ptr(), x.len() as u64) }).unwrap());
            x
        }
        /// L in CSC, its unit diagonal not stored.
        pub fn l(&self) -> CsMatI<f64, usize> {
            self.valid();
            let (n, nnz) = (self.sym.n, self.nnz());
            let (mut ip, mut ind, mut data) = (vec![0u32; n + 1], vec![0u32; nnz], vec![0.0; nnz]);
            CTX.with(|c| check(c.0, unsafe {
                ffi::sprs_b200_ldl_get_l(self.h.0, ip.as_mut_ptr(), ind.as_mut_ptr(), data.as_mut_ptr()) }).unwrap());
            CsMatI::new_csc((n, n), ip.into_iter().map(|v| v as usize).collect(),
                            ind.into_iter().map(|v| v as usize).collect(), data)
        }
        pub fn d(&self) -> Vec<f64> {
            self.valid();
            let mut d = vec![0.0; self.sym.n];
            CTX.with(|c| check(c.0, unsafe { ffi::sprs_b200_ldl_get_d(self.h.0, d.as_mut_ptr(), d.len() as u64) }).unwrap());
            d
        }
        pub fn problem_size(&self) -> usize { self.sym.n }
        pub fn nnz(&self) -> usize { self.sym.nnz() }
    }
}
