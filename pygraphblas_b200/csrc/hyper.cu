// hyper.cu -- hypersparse operands of GrB_mxm / GrB_mxv / GrB_vxm.
//
// The reference's idiomatic unsized objects are 2^60 x 2^60 (reference: pygraphblas/matrix.py:167-170,
// vector.py:250-286; SuiteSparse keeps them hypersparse).  In HBM the kernels index rows and columns with 32 bits, so an
// object whose dimension exceeds 2^31-1 is held as sorted tuples and computed on in its COMPACT index space:
//
//     rows  = the sorted distinct row ids that occur in op(A), w / C and the mask        (the "row-id list")
//     cols  = likewise for the inner / column dimension
//     op(A), u, w, mask  ->  the same entries renumbered by rank in those lists: a CSR over the non-empty rows only
//
// Positions outside the lists hold no entry in any operand, so the product, the accumulator and the mask (value,
// structural, complemented) and GrB_REPLACE act on them exactly as on nothing: the result computed on the compact
// objects and renumbered back IS the result on the 2^60 space.  The arithmetic runs through the same CUDA kernels
// (GrB_mxv / GrB_mxm on the compact handles); only the renumbering of call arguments happens on the host, where the
// tuples of such objects live anyway.  Nothing is computed on the host.
#include "common.cuh"
#include <algorithm>
#include <vector>
#include <string.h>

static const uint64_t HYPER_DIM = ((uint64_t)1 << 31) - 1;

extern "C" GrB_Info GrB_Matrix_new(GrB_Matrix *A, GrB_Type type, GrB_Index nrows, GrB_Index ncols);
extern "C" GrB_Info GrB_Matrix_free(GrB_Matrix *A);
extern "C" GrB_Info GrB_Vector_new(GrB_Vector *v, GrB_Type type, GrB_Index n);
extern "C" GrB_Info GrB_Vector_free(GrB_Vector *v);
extern "C" GrB_Info GrB_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Vector u, const GrB_Descriptor d);
extern "C" GrB_Info GrB_vxm(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Vector u, const GrB_Matrix A, const GrB_Descriptor d);
extern "C" GrB_Info GrB_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Matrix B, const GrB_Descriptor d);

bool gb_hyper_matrix(const GrB_Matrix A) { return A && (A->nrows > HYPER_DIM || A->ncols > HYPER_DIM); }
bool gb_hyper_vector(const GrB_Vector v) { return v && v->n > HYPER_DIM; }

typedef std::vector<uint64_t> Ids;
static void ids_finish(Ids &s) { std::sort(s.begin(), s.end()); s.erase(std::unique(s.begin(), s.end()), s.end()); }
static inline uint64_t rank_of(const Ids &s, uint64_t id) { return (uint64_t)(std::lower_bound(s.begin(), s.end(), id) - s.begin()); }

// a compact copy of v over the id list `ids` (every id of v is in the list)
static GrB_Info compact_vector(const GrB_Vector v, const Ids &ids, GrB_Vector *out) {
    GB_TRY(GrB_Vector_new(out, v->type, (GrB_Index)ids.size()));
    GrB_Vector c = *out;
    c->hi.resize(v->hi.size()); c->hx = v->hx;
    for (size_t k = 0; k < v->hi.size(); ++k) c->hi[k] = rank_of(ids, v->hi[k]);      // order is preserved: ranks are monotone
    c->host_valid = true;
    return GrB_SUCCESS;
}
// a compact copy of A: rows renumbered by `rows`, columns by `cols`
static GrB_Info compact_matrix(const GrB_Matrix A, const Ids &rows, const Ids &cols, GrB_Matrix *out) {
    GB_TRY(GrB_Matrix_new(out, A->type, (GrB_Index)rows.size(), (GrB_Index)cols.size()));
    GrB_Matrix c = *out;
    const size_t n = A->hi.size();
    c->hi.resize(n); c->hj.resize(n); c->hx = A->hx;
    for (size_t k = 0; k < n; ++k) { c->hi[k] = rank_of(rows, A->hi[k]); c->hj[k] = rank_of(cols, A->hj[k]); }    // row-major order is preserved
    c->host_valid = true;
    return GrB_SUCCESS;
}
// the result of a compact call, renumbered back into w (dimension unchanged)
static GrB_Info expand_vector(GrB_Vector w, GrB_Vector c, const Ids &ids) {
    GB_TRY(vector_ensure_host(c));
    vector_invalidate_device(w);
    w->hi.resize(c->hi.size()); w->hx = c->hx; w->pi.clear(); w->px.clear();
    for (size_t k = 0; k < c->hi.size(); ++k) w->hi[k] = ids[c->hi[k]];
    w->host_valid = true;
    return GrB_SUCCESS;
}
static GrB_Info expand_matrix(GrB_Matrix C, GrB_Matrix c, const Ids &rows, const Ids &cols) {
    GB_TRY(matrix_ensure_host(c));
    matrix_invalidate_device(C);
    const size_t n = c->hi.size();
    C->hi.resize(n); C->hj.resize(n); C->hx = c->hx; C->pi.clear(); C->pj.clear(); C->px.clear();
    for (size_t k = 0; k < n; ++k) { C->hi[k] = rows[c->hi[k]]; C->hj[k] = cols[c->hj[k]]; }
    C->host_valid = true;
    return GrB_SUCCESS;
}

// w<mask> = accum(w, op(A) u)  (vxm == false)   /   w'<mask'> = accum(w', u' op(A))  (vxm == true), some operand beyond 2^31-1
GrB_Info hyper_mxv(GrB_Vector w, const GrB_Vector mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Vector u,
                   const GrB_Descriptor desc, bool vxm) {
    const DescFlags f = desc_flags(desc);
    const bool tran = vxm ? !f.tran1 : f.tran0;                 // the output runs along A's columns when true
    const char *fn = vxm ? "GrB_vxm" : "GrB_mxv";
    const uint64_t out_n = tran ? A->ncols : A->nrows, in_n = tran ? A->nrows : A->ncols;
    if (u->n != in_n || w->n != out_n || (mask && mask->n != out_n)) return gb_fail(GrB_DIMENSION_MISMATCH, &w->err, "%s: dimensions do not match", fn);
    if (!G.have_device) return gb_fail(GrB_PANIC, &w->err, "%s: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)", fn);
    GB_TRY(matrix_ensure_host(A)); GB_TRY(vector_ensure_host(u)); GB_TRY(vector_ensure_host(w));
    if (mask) GB_TRY(vector_ensure_host(mask));
    // row-id and column-id lists of A (as stored); the vectors join the list of the side they run along
    Ids rows(A->hi), cols(A->hj);
    Ids &out_ids = tran ? cols : rows, &in_ids = tran ? rows : cols;
    out_ids.insert(out_ids.end(), w->hi.begin(), w->hi.end());
    if (mask) out_ids.insert(out_ids.end(), mask->hi.begin(), mask->hi.end());
    in_ids.insert(in_ids.end(), u->hi.begin(), u->hi.end());
    ids_finish(rows); ids_finish(cols);
    if (rows.size() > HYPER_DIM || cols.size() > HYPER_DIM) return gb_fail(GrB_INVALID_VALUE, &w->err, "%s: more than 2^31-1 non-empty rows or columns", fn);
    if (rows.empty()) rows.push_back(0);                         // keep the compact objects non-degenerate
    if (cols.empty()) cols.push_back(0);
    GrB_Matrix Ac = nullptr; GrB_Vector uc = nullptr, wc = nullptr, mc = nullptr;
    GrB_Info r = compact_matrix(A, rows, cols, &Ac);
    if (r == GrB_SUCCESS) r = compact_vector(u, in_ids, &uc);
    if (r == GrB_SUCCESS) r = compact_vector(w, out_ids, &wc);
    if (r == GrB_SUCCESS && mask) r = compact_vector(mask, out_ids, &mc);
    if (r == GrB_SUCCESS && op_is_positional(s->mul->opcode)) {
        // a positional multiply returns original indices, not compact ranks: the id lists go to the device
        DevBuf<uint64_t> din, dout;
        r = upload_indices(in_ids, din, &w->err);
        if (r == GrB_SUCCESS) r = upload_indices(out_ids, dout, &w->err);
        if (r == GrB_SUCCESS) r = positional_mxv(wc, mc, accum, s, Ac, uc, f, vxm, din, dout);
    } else if (r == GrB_SUCCESS) r = vxm ? GrB_vxm(wc, mc, accum, s, uc, Ac, desc) : GrB_mxv(wc, mc, accum, s, Ac, uc, desc);
    if (r == GrB_SUCCESS) r = expand_vector(w, wc, out_ids);
    else if (wc) w->err = wc->err;
    GrB_Matrix_free(&Ac); GrB_Vector_free(&uc); GrB_Vector_free(&wc); GrB_Vector_free(&mc);
    return r;
}

// C<Mask> = accum(C, op(A) op(B)), some operand beyond 2^31-1
GrB_Info hyper_mxm(GrB_Matrix C, const GrB_Matrix Mask, const GrB_BinaryOp accum, const GrB_Semiring s, const GrB_Matrix A, const GrB_Matrix B,
                   const GrB_Descriptor desc) {
    const DescFlags f = desc_flags(desc);
    const uint64_t am = f.tran0 ? A->ncols : A->nrows, ak = f.tran0 ? A->nrows : A->ncols;
    const uint64_t bk = f.tran1 ? B->ncols : B->nrows, bn = f.tran1 ? B->nrows : B->ncols;
    if (ak != bk || C->nrows != am || C->ncols != bn || (Mask && (Mask->nrows != am || Mask->ncols != bn)))
        return gb_fail(GrB_DIMENSION_MISMATCH, &C->err, "GrB_mxm: dimensions do not match");
    if (!G.have_device) return gb_fail(GrB_PANIC, &C->err, "GrB_mxm: no CUDA device: libb200grb computes only on the GPU (no CPU fallback)");
    GB_TRY(matrix_ensure_host(A)); GB_TRY(matrix_ensure_host(B)); GB_TRY(matrix_ensure_host(C));
    if (Mask) GB_TRY(matrix_ensure_host(Mask));
    // three index spaces: m (rows of op(A), C, Mask), k (inner), n (columns of op(B), C, Mask)
    Ids ms(f.tran0 ? A->hj : A->hi), ks(f.tran0 ? A->hi : A->hj), ns(f.tran1 ? B->hi : B->hj);
    const Ids &bks = f.tran1 ? B->hj : B->hi;
    ks.insert(ks.end(), bks.begin(), bks.end());
    ms.insert(ms.end(), C->hi.begin(), C->hi.end()); ns.insert(ns.end(), C->hj.begin(), C->hj.end());
    if (Mask) { ms.insert(ms.end(), Mask->hi.begin(), Mask->hi.end()); ns.insert(ns.end(), Mask->hj.begin(), Mask->hj.end()); }
    ids_finish(ms); ids_finish(ks); ids_finish(ns);
    if (ms.size() > HYPER_DIM || ks.size() > HYPER_DIM || ns.size() > HYPER_DIM) return gb_fail(GrB_INVALID_VALUE, &C->err, "GrB_mxm: more than 2^31-1 non-empty rows or columns");
    if (ms.empty()) ms.push_back(0);
    if (ks.empty()) ks.push_back(0);
    if (ns.empty()) ns.push_back(0);
    GrB_Matrix Ac = nullptr, Bc = nullptr, Cc = nullptr, Mc = nullptr;
    GrB_Info r = f.tran0 ? compact_matrix(A, ks, ms, &Ac) : compact_matrix(A, ms, ks, &Ac);
    if (r == GrB_SUCCESS) r = f.tran1 ? compact_matrix(B, ns, ks, &Bc) : compact_matrix(B, ks, ns, &Bc);
    // C may alias A or B: the compact C is a separate object either way, the result replaces C at the end
    if (r == GrB_SUCCESS) r = compact_matrix(C, ms, ns, &Cc);
    if (r == GrB_SUCCESS && Mask) r = compact_matrix(Mask, ms, ns, &Mc);
    if (r == GrB_SUCCESS && op_is_positional(s->mul->opcode)) {
        DevBuf<uint64_t> dm, dk, dn;
        r = upload_indices(ms, dm, &C->err);
        if (r == GrB_SUCCESS) r = upload_indices(ks, dk, &C->err);
        if (r == GrB_SUCCESS) r = upload_indices(ns, dn, &C->err);
        if (r == GrB_SUCCESS) r = positional_mxm(Cc, Mc, accum, s, Ac, Bc, f, dm, dk, dn);
    } else if (r == GrB_SUCCESS) r = GrB_mxm(Cc, Mc, accum, s, Ac, Bc, desc);
    if (r == GrB_SUCCESS) r = expand_matrix(C, Cc, ms, ns);
    else if (Cc) C->err = Cc->err;
    GrB_Matrix_free(&Ac); GrB_Matrix_free(&Bc); GrB_Matrix_free(&Cc); GrB_Matrix_free(&Mc);
    return r;
}
