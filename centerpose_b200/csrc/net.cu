// Op-program entry points of the C ABI: validation, the choice of each tensor-core op's kernel family, dispatch.
#include "tc_common.cuh"

namespace cpb {
int run_op_simt_dispatch(const cpb200_op &op, cudaStream_t st);
bool simt_runs_split(int type);
int heads_prepare(const cpb200_op &op, Prepared **out);
int heads_run(const Prepared &p, const cpb200_op &op, cudaStream_t st);
bool stem_tc_eligible(const cpb200_op &op);
int stem_tc_run(const cpb200_op &op, cudaStream_t st);
bool sp_eligible(const cpb200_op &op);
int sp_run(const cpb200_op &op, cudaStream_t st);
bool c3_eligible(const cpb200_op &op);
int c3_prepare(const cpb200_op &op, Prepared **out);
int c3_run(const Prepared &p, const cpb200_op &op, cudaStream_t st);
int tap_prepare(const cpb200_op &op, Prepared **out);
int tap_run(const Prepared &p, const cpb200_op &op, cudaStream_t st);
}  // namespace cpb

static int validate(const cpb200_op &op, int i) {
  if (op.B <= 0 || op.H <= 0 || op.W <= 0 || op.Ho <= 0 || op.Wo <= 0)
    return cpb::fail(CPB200_ERR_ARG, "op %d: bad shape", i);
  if (op.nsrc < 1 || op.nsrc > 4) return cpb::fail(CPB200_ERR_ARG, "op %d: nsrc %d", i, op.nsrc);
  for (int s = 0; s < op.nsrc; ++s)
    if (!op.src[s] || op.cin[s] <= 0) return cpb::fail(CPB200_ERR_ARG, "op %d: null/empty input %d", i, s);
  if (!op.dst && op.type != CPB200_OP_HEADS) return cpb::fail(CPB200_ERR_ARG, "op %d: null dst", i);   // HEADS: per-head dst
  if (op.act_dtype < CPB200_F32 || op.act_dtype > CPB200_F16X2)
    return cpb::fail(CPB200_ERR_ARG, "op %d: bad act_dtype", i);
  if ((op.act_dtype == CPB200_BF16X2 || op.act_dtype == CPB200_F16X2) && !(op.flags & CPB200_FLAG_TC) && !cpb::simt_runs_split(op.type))
    return cpb::fail(CPB200_ERR_ARG, "op %d: split-precision activations need the tensor-core path (or an element-wise op / CONVERT)", i);
  if ((op.type == CPB200_OP_CONV || op.type == CPB200_OP_DCN || op.type == CPB200_OP_STEM || op.type == CPB200_OP_HEADS) && !op.weight)
    return cpb::fail(CPB200_ERR_ARG, "op %d: null weight", i);
  for (int s = 0; s < op.nsrc; ++s)
    if (op.src_pitch[s] != 0 && (op.src_pitch[s] < op.cin[s] || (op.type != CPB200_OP_CONV && op.src_pitch[s] != op.cin[s])))
      return cpb::fail(CPB200_ERR_ARG, "op %d: channel-slice inputs (src_pitch) are supported by CONV ops only", i);
  if (op.out_sy < 1 || op.out_sx < 1 || op.Hd < 1 || op.Wd < 1)
    return cpb::fail(CPB200_ERR_ARG, "op %d: bad output mapping", i);
  return CPB200_OK;
}

// The kernel family of an op flagged CPB200_FLAG_TC (tc_common.cuh: Route).
static int prepare_tc(const cpb200_op &op, int i, cpb::Prepared **out) {
  using cpb::Route;
  if (op.type == CPB200_OP_HEADS) return cpb::heads_prepare(op, out);
  if (op.type == CPB200_OP_STEM) {
    if (!cpb::stem_tc_eligible(op))
      return cpb::fail(CPB200_ERR_ARG, "op %d: the tensor-core stem needs 7x7 / pad 3, Cin 3, stride 1 or 2, cout 16 or 64 "
                                       "(split precisions: stride 1)", i);
    *out = new cpb::Prepared(Route::STEM);
    return CPB200_OK;
  }
  if (cpb::sp_eligible(op)) {       // small-channel 3x3 conv: the SIMT-fed wgmma kernel
    *out = new cpb::Prepared(Route::SP);
    return CPB200_OK;
  }
  if (cpb::c3_eligible(op)) return cpb::c3_prepare(op, out);
  return cpb::tap_prepare(op, out);
}

extern "C" size_t cpb200_sizeof_op(void) { return sizeof(cpb200_op); }

extern "C" int cpb200_prepare_ops(cpb200_op *ops, int n) {
  if (!ops || n < 0) return cpb::fail(CPB200_ERR_ARG, "prepare_ops: bad arguments");
  for (int i = 0; i < n; ++i) {
    if (int rc = validate(ops[i], i)) return rc;
    cpb::Prepared *p = nullptr;
    if (ops[i].flags & CPB200_FLAG_TC) {
      if (int rc = prepare_tc(ops[i], i, &p)) return rc;
    } else if (ops[i].type == CPB200_OP_HEADS) {
      return cpb::fail(CPB200_ERR_ARG, "op %d: HEADS runs on the tensor-core path only", i);
    }
    ops[i].tc = p;
  }
  return CPB200_OK;
}

extern "C" int cpb200_release_ops(cpb200_op *ops, int n) {
  if (!ops) return CPB200_OK;
  for (int i = 0; i < n; ++i) {
    delete static_cast<cpb::Prepared *>(ops[i].tc);
    ops[i].tc = nullptr;
  }
  return CPB200_OK;
}

extern "C" int cpb200_run_ops(const cpb200_op *ops, int n, void *stream) {
  if (!ops || n < 0) return cpb::fail(CPB200_ERR_ARG, "run_ops: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  using cpb::Route;
  for (int i = 0; i < n; ++i) {
    const cpb200_op &op = ops[i];
    const cpb::Prepared *p = static_cast<const cpb::Prepared *>(op.tc);
    int rc = CPB200_OK;
    if (!p) {
      if (op.flags & CPB200_FLAG_TC) return cpb::fail(CPB200_ERR_STATE, "op %d: tensor-core op not prepared", i);
      rc = cpb::run_op_simt_dispatch(op, st);
    } else {
      switch (p->route) {
        case Route::HEADS: rc = cpb::heads_run(*p, op, st); break;
        case Route::STEM: rc = cpb::stem_tc_run(op, st); break;
        case Route::SP: rc = cpb::sp_run(op, st); break;
        case Route::HALO: rc = cpb::c3_run(*p, op, st); break;
        case Route::TAP: rc = cpb::tap_run(*p, op, st); break;
      }
    }
    if (rc) return rc;
  }
  return CPB200_OK;
}
