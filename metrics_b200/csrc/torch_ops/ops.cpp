// torch.ops.metrics_b200.* — the hot-path entry points registered as PyTorch operators (TORCH_LIBRARY schemas, SURVEY.md
// §8(b) "what a C-ABI replacement must export").  Every operator is a thin shim: it checks devices / dtypes / contiguity the
// way the dispatcher cannot, takes raw pointers and the CURRENT CUDA stream, and calls the plain-C ABI of
// include/metrics_b200.h (libmetrics_b200.so, hand-written sm_90a kernels) — no arithmetic happens here.  Registered for the
// CUDA dispatch key only: there is no CPU implementation.  Shape-only ("fake") implementations for tracing are registered
// from Python (metrics_b200/torch_ops.py).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <ATen/ATen.h>
#include <torch/library.h>

#include "../../../include/metrics_b200.h"

namespace {

int dtype_tag(const at::Tensor& t) {
    switch (t.scalar_type()) {
        case at::kFloat: return MB200_F32;
        case at::kHalf: return MB200_F16;
        case at::kBFloat16: return MB200_BF16;
        case at::kDouble: return MB200_F64;
        case at::kLong: return MB200_I64;
        case at::kInt: return MB200_I32;
        case at::kShort: return MB200_I16;
        case at::kChar: return MB200_I8;
        case at::kByte: return MB200_U8;
        case at::kBool: return MB200_BOOL;
        default: TORCH_CHECK(false, "metrics_b200: unsupported tensor dtype ", t.scalar_type());
    }
}

void ok(int rc, const char* what) {
    if (rc == MB200_OK) return;
    const char* msg = mb200_last_error();
    TORCH_CHECK_VALUE(rc != MB200_ERR_INVALID, "metrics_b200.", what, ": ", msg);
    TORCH_CHECK(false, "metrics_b200.", what, " failed (code ", rc, "): ", msg);
}

void* stream_of(const at::Tensor& t) { return at::cuda::getCurrentCUDAStream(t.get_device()).stream(); }

void same_cuda(const at::Tensor& a, std::initializer_list<const at::Tensor*> others) {
    TORCH_CHECK(a.is_cuda(), "metrics_b200 kernels only run on CUDA tensors (sm_90a): there is no CPU fallback");
    for (const at::Tensor* o : others)
        TORCH_CHECK(o->device() == a.device(), "Expected all tensors to be on the same device, but found at least two devices, ",
                    a.device(), " and ", o->device(), "!");
}

uint32_t* flag_ptr(const c10::optional<at::Tensor>& f) {
    if (!f.has_value()) return nullptr;
    TORCH_CHECK(f->scalar_type() == at::kInt && f->numel() >= 1, "err_flag must be an int32 tensor");
    return reinterpret_cast<uint32_t*>(f->data_ptr());
}

// confusion_matrix.py:297-328 + classification/confusion_matrix.py:286
void confmat_update_(at::Tensor& confmat, const at::Tensor& preds, const at::Tensor& target, int64_t num_classes,
                     c10::optional<int64_t> ignore_index, const c10::optional<at::Tensor>& err_flag) {
    same_cuda(confmat, {&preds, &target});
    TORCH_CHECK(confmat.scalar_type() == at::kLong && confmat.is_contiguous() && confmat.numel() == num_classes * num_classes,
                "confmat must be a contiguous int64 [C, C] tensor");
    const c10::cuda::CUDAGuard guard(confmat.device());
    const at::Tensor p = preds.contiguous(), t = target.contiguous();
    const bool has_class_dim = p.dim() == t.dim() + 1;
    int64_t n_outer = p.numel(), inner = 1;
    if (has_class_dim) {
        n_outer = p.size(0);
        for (int64_t d = 2; d < p.dim(); ++d) inner *= p.size(d);
    }
    ok(mb200_multiclass_confmat_update(p.data_ptr(), dtype_tag(p), has_class_dim, t.data_ptr(), dtype_tag(t), n_outer, num_classes,
                                       inner, ignore_index.has_value(), ignore_index.value_or(0), confmat.data_ptr<int64_t>(),
                                       flag_ptr(err_flag), stream_of(confmat)),
       "confmat_update_");
}

// stat_scores.py:328-448 + classification/stat_scores.py:69-80
void stat_scores_update_(at::Tensor& tp, at::Tensor& fp, at::Tensor& tn, at::Tensor& fn, at::Tensor& workspace,
                         const at::Tensor& preds, const at::Tensor& target, int64_t num_classes,
                         c10::optional<int64_t> ignore_index, bool micro, const c10::optional<at::Tensor>& err_flag) {
    same_cuda(tp, {&fp, &tn, &fn, &workspace, &preds, &target});
    for (const at::Tensor* s : {&tp, &fp, &tn, &fn, &workspace})
        TORCH_CHECK(s->scalar_type() == at::kLong && s->is_contiguous(), "states and workspace must be contiguous int64 tensors");
    TORCH_CHECK(workspace.numel() >= 3 * num_classes + 2, "workspace needs 3 * num_classes + 2 int64 words");
    const c10::cuda::CUDAGuard guard(tp.device());
    const at::Tensor p = preds.contiguous(), t = target.contiguous();
    const bool has_class_dim = p.dim() == t.dim() + 1;
    int64_t n_outer = p.numel(), inner = 1;
    if (has_class_dim) {
        n_outer = p.size(0);
        for (int64_t d = 2; d < p.dim(); ++d) inner *= p.size(d);
    }
    ok(mb200_multiclass_stat_scores_update(p.data_ptr(), dtype_tag(p), has_class_dim, t.data_ptr(), dtype_tag(t), n_outer,
                                           num_classes, inner, ignore_index.has_value(), ignore_index.value_or(0), micro,
                                           tp.data_ptr<int64_t>(), fp.data_ptr<int64_t>(), tn.data_ptr<int64_t>(),
                                           fn.data_ptr<int64_t>(), workspace.data_ptr<int64_t>(), flag_ptr(err_flag), stream_of(tp)),
       "stat_scores_update_");
}

// K11: collections.py:231-262 fan-out fused
at::Tensor stats_softmax_update_(at::Tensor& tp, at::Tensor& fp, at::Tensor& tn, at::Tensor& fn, at::Tensor& workspace,
                                 const at::Tensor& preds, const at::Tensor& target, int64_t num_classes, bool micro,
                                 const c10::optional<at::Tensor>& err_flag) {
    same_cuda(tp, {&fp, &tn, &fn, &workspace, &preds, &target});
    TORCH_CHECK(preds.dim() == 2 && target.dim() == 1 && preds.size(0) == target.size(0) && preds.size(1) == num_classes,
                "preds must be [N, num_classes] and target [N]");
    const c10::cuda::CUDAGuard guard(tp.device());
    const at::Tensor p = preds.contiguous(), t = target.contiguous();
    at::Tensor probs = at::empty_like(p);
    at::Tensor flag = at::empty({1}, p.options().dtype(at::kInt));
    ok(mb200_multiclass_stats_softmax_update(p.data_ptr(), dtype_tag(p), t.data_ptr(), dtype_tag(t), p.size(0), num_classes, micro,
                                             tp.data_ptr<int64_t>(), fp.data_ptr<int64_t>(), tn.data_ptr<int64_t>(),
                                             fn.data_ptr<int64_t>(), workspace.data_ptr<int64_t>(), probs.data_ptr(),
                                             reinterpret_cast<uint32_t*>(flag.data_ptr()), flag_ptr(err_flag), stream_of(tp)),
       "stats_softmax_update_");
    return probs;
}

// utilities/compute.py:190-229
at::Tensor normalize_logits_if_needed(const at::Tensor& preds, const std::string& normalization) {
    same_cuda(preds, {});
    const c10::cuda::CUDAGuard guard(preds.device());
    const at::Tensor p = preds.contiguous();
    at::Tensor out = at::empty_like(p);
    if (p.numel() == 0) return out;
    at::Tensor flag = at::empty({1}, p.options().dtype(at::kInt));
    uint32_t* f = reinterpret_cast<uint32_t*>(flag.data_ptr());
    if (normalization == "sigmoid") {
        ok(mb200_curve_sigmoid_if_logits(p.data_ptr(), dtype_tag(p), p.numel(), out.data_ptr(), f, stream_of(p)), "sigmoid_if_logits");
    } else {
        TORCH_CHECK_VALUE(normalization == "softmax" && p.dim() == 2, "softmax normalisation expects an [N, C] tensor");
        ok(mb200_curve_softmax_if_logits(p.data_ptr(), dtype_tag(p), p.size(0), p.size(1), out.data_ptr(), f, stream_of(p)),
           "softmax_if_logits");
    }
    return out;
}

// precision_recall_curve.py:30-82 (+ roc.py / auroc.py / average_precision.py scalars) for num_classes one-vs-rest curves
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> curve_evaluate(
    const at::Tensor& preds, const at::Tensor& target, int64_t num_classes, int64_t pos_label, bool want_curve) {
    same_cuda(preds, {&target});
    const c10::cuda::CUDAGuard guard(preds.device());
    const at::Tensor p = preds.contiguous(), t = target.contiguous();
    const int64_t n = t.numel();
    const auto f32 = p.options().dtype(at::kFloat);
    at::Tensor ws = at::empty({mb200_curve_workspace_bytes_for(num_classes, n, dtype_tag(p))}, p.options().dtype(at::kByte));
    at::Tensor auroc = at::empty({num_classes}, f32), ap = at::empty({num_classes}, f32);
    at::Tensor counts = at::empty({num_classes, 3}, p.options().dtype(at::kLong));
    const int64_t cn = want_curve ? n : 0;
    at::Tensor fps = at::empty({num_classes, cn}, f32), tps = at::empty({num_classes, cn}, f32);
    at::Tensor thr = at::empty({num_classes, cn}, p.scalar_type() == at::kDouble ? p.options() : f32);
    ok(mb200_curve_evaluate(p.data_ptr(), dtype_tag(p), t.data_ptr(), dtype_tag(t), n, num_classes, pos_label, ws.data_ptr(),
                            ws.numel(), auroc.data_ptr<float>(), ap.data_ptr<float>(), counts.data_ptr<int64_t>(),
                            want_curve ? fps.data_ptr<float>() : nullptr, want_curve ? tps.data_ptr<float>() : nullptr,
                            want_curve ? thr.data_ptr() : nullptr, nullptr, stream_of(p)),
       "curve_evaluate");
    return {auroc, ap, counts, fps, tps, thr};
}

// precision_recall_curve.py:191-251, 464-533, 745-799; thresholds ascending, of any float or integer dtype
void binned_curve_update_(at::Tensor& confmat, at::Tensor& scratch, const at::Tensor& preds, const at::Tensor& target,
                          const at::Tensor& thresholds, int64_t num_classes, bool multilabel, c10::optional<int64_t> ignore_index) {
    same_cuda(confmat, {&scratch, &preds, &target, &thresholds});
    TORCH_CHECK(confmat.scalar_type() == at::kLong && confmat.is_contiguous() && scratch.scalar_type() == at::kLong &&
                    thresholds.is_contiguous(),
                "confmat / scratch must be int64, all contiguous");
    TORCH_CHECK(scratch.numel() >= mb200_binned_curve_scratch_words(num_classes, thresholds.numel()), "scratch too small");
    const c10::cuda::CUDAGuard guard(confmat.device());
    const at::Tensor p = preds.contiguous(), t = target.contiguous();
    const int64_t n = multilabel || num_classes == 1 ? (num_classes == 1 ? p.numel() : p.size(0)) : p.size(0);
    const int thr_tag = dtype_tag(thresholds);
    const int cmp = mb200_binned_curve_compare_dtype(dtype_tag(p), thr_tag, n, num_classes, multilabel ? 1 : 0);
    const int rc = multilabel
        ? mb200_binned_curve_update_multilabel(p.data_ptr(), dtype_tag(p), t.data_ptr(), dtype_tag(t), n, num_classes,
                                               thresholds.data_ptr(), thr_tag, cmp, thresholds.numel(), ignore_index.has_value(),
                                               ignore_index.value_or(0), confmat.data_ptr<int64_t>(),
                                               reinterpret_cast<uint64_t*>(scratch.data_ptr()), stream_of(confmat))
        : mb200_binned_curve_update(p.data_ptr(), dtype_tag(p), t.data_ptr(), dtype_tag(t), n, num_classes, thresholds.data_ptr(),
                                    thr_tag, cmp, thresholds.numel(), confmat.data_ptr<int64_t>(),
                                    reinterpret_cast<uint64_t*>(scratch.data_ptr()), stream_of(confmat));
    ok(rc, "binned_curve_update_");
}

// functional/regression/*.py `_x_update`: float64 [num_sums, num_outputs]
at::Tensor regression_sums(const at::Tensor& preds, const at::Tensor& target, int64_t op, int64_t num_outputs, double param, double eps) {
    same_cuda(preds, {&target});
    TORCH_CHECK(preds.scalar_type() == target.scalar_type() && preds.numel() == target.numel(), "preds / target must match");
    const c10::cuda::CUDAGuard guard(preds.device());
    const at::Tensor p = preds.contiguous(), t = target.contiguous();
    const int k = mb200_regression_num_sums((int)op);
    TORCH_CHECK_VALUE(k > 0, "unknown regression op ", op);
    const int64_t n = p.numel() / num_outputs;
    at::Tensor out = at::empty({k, num_outputs}, p.options().dtype(at::kDouble));
    at::Tensor scratch = at::empty({mb200_regression_scratch_doubles(n, num_outputs, (int)op)}, out.options());
    ok(mb200_regression_sums(p.data_ptr(), t.data_ptr(), dtype_tag(p), n, num_outputs, (int)op, param, eps, out.data_ptr<double>(),
                             scratch.data_ptr<double>(), stream_of(p)),
       "regression_sums");
    return out;
}

}  // namespace

TORCH_LIBRARY(metrics_b200, m) {
    m.def("confmat_update_(Tensor(a!) confmat, Tensor preds, Tensor target, int num_classes, int? ignore_index=None, "
          "Tensor? err_flag=None) -> ()");
    m.def("stat_scores_update_(Tensor(a!) tp, Tensor(b!) fp, Tensor(c!) tn, Tensor(d!) fn, Tensor(e!) workspace, Tensor preds, "
          "Tensor target, int num_classes, int? ignore_index=None, bool micro=False, Tensor? err_flag=None) -> ()");
    m.def("stats_softmax_update_(Tensor(a!) tp, Tensor(b!) fp, Tensor(c!) tn, Tensor(d!) fn, Tensor(e!) workspace, Tensor preds, "
          "Tensor target, int num_classes, bool micro=False, Tensor? err_flag=None) -> Tensor");
    m.def("normalize_logits_if_needed(Tensor preds, str normalization) -> Tensor");
    m.def("curve_evaluate(Tensor preds, Tensor target, int num_classes=1, int pos_label=1, bool want_curve=False) -> "
          "(Tensor auroc, Tensor ap, Tensor counts, Tensor fps, Tensor tps, Tensor thresholds)");
    m.def("binned_curve_update_(Tensor(a!) confmat, Tensor(b!) scratch, Tensor preds, Tensor target, Tensor thresholds, "
          "int num_classes=1, bool multilabel=False, int? ignore_index=None) -> ()");
    m.def("regression_sums(Tensor preds, Tensor target, int op, int num_outputs=1, float param=0.0, float eps=0.0) -> Tensor");
}

TORCH_LIBRARY_IMPL(metrics_b200, CUDA, m) {
    m.impl("confmat_update_", &confmat_update_);
    m.impl("stat_scores_update_", &stat_scores_update_);
    m.impl("stats_softmax_update_", &stats_softmax_update_);
    m.impl("normalize_logits_if_needed", &normalize_logits_if_needed);
    m.impl("curve_evaluate", &curve_evaluate);
    m.impl("binned_curve_update_", &binned_curve_update_);
    m.impl("regression_sums", &regression_sums);
}
