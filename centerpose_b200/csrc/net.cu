// Op-program entry points of the C ABI: validation, tensor-core preparation, dispatch.
#include "common.cuh"

namespace cpb {
int run_op_simt_dispatch(const cpb200_op &op, cudaStream_t st);
int tc_prepare_op(cpb200_op &op);
int tc_release_op(cpb200_op &op);
int tc_run_op(const cpb200_op &op, cudaStream_t st);
bool sp_eligible(const cpb200_op &op);
int sp_run(const cpb200_op &op, cudaStream_t st);
bool stem_tc_eligible(const cpb200_op &op);
int stem_tc_run(const cpb200_op &op, cudaStream_t st);
}  // namespace cpb

static int validate(const cpb200_op &op, int i) {
  if (op.B <= 0 || op.H <= 0 || op.W <= 0 || op.Ho <= 0 || op.Wo <= 0)
    return cpb::fail(CPB200_ERR_ARG, "op %d: bad shape", i);
  if (op.nsrc < 1 || op.nsrc > 4) return cpb::fail(CPB200_ERR_ARG, "op %d: nsrc %d", i, op.nsrc);
  for (int s = 0; s < op.nsrc; ++s)
    if (!op.src[s] || op.cin[s] <= 0) return cpb::fail(CPB200_ERR_ARG, "op %d: null/empty input %d", i, s);
  if (!op.dst) return cpb::fail(CPB200_ERR_ARG, "op %d: null dst", i);
  if (op.act_dtype < CPB200_F32 || op.act_dtype > CPB200_F16X2)
    return cpb::fail(CPB200_ERR_ARG, "op %d: bad act_dtype", i);
  if ((op.act_dtype == CPB200_BF16X2 || op.act_dtype == CPB200_F16X2) && !(op.flags & CPB200_FLAG_TC) &&
      op.type != CPB200_OP_CONVERT && op.type != CPB200_OP_MAXPOOL && op.type != CPB200_OP_DWDECONV_ADD &&
      op.type != CPB200_OP_DWCONV && op.type != CPB200_OP_AVGPOOL && op.type != CPB200_OP_SCALE_ADD && op.type != CPB200_OP_UPSAMPLE_ADD &&
      op.type != CPB200_OP_S2D)
    return cpb::fail(CPB200_ERR_ARG, "op %d: split-precision activations need the tensor-core path (or an element-wise op / CONVERT)", i);
  if ((op.type == CPB200_OP_CONV || op.type == CPB200_OP_DCN || op.type == CPB200_OP_STEM) && !op.weight)
    return cpb::fail(CPB200_ERR_ARG, "op %d: null weight", i);
  for (int s = 0; s < op.nsrc; ++s)
    if (op.src_pitch[s] != 0 && (op.src_pitch[s] < op.cin[s] || (op.type != CPB200_OP_CONV && op.src_pitch[s] != op.cin[s])))
      return cpb::fail(CPB200_ERR_ARG, "op %d: channel-slice inputs (src_pitch) are supported by CONV ops only", i);
  if (op.out_sy < 1 || op.out_sx < 1 || op.Hd < 1 || op.Wd < 1)
    return cpb::fail(CPB200_ERR_ARG, "op %d: bad output mapping", i);
  return CPB200_OK;
}

extern "C" size_t cpb200_sizeof_op(void) { return sizeof(cpb200_op); }

extern "C" int cpb200_prepare_ops(cpb200_op *ops, int n) {
  if (!ops || n < 0) return cpb::fail(CPB200_ERR_ARG, "prepare_ops: bad arguments");
  for (int i = 0; i < n; ++i) {
    int rc = validate(ops[i], i);
    if (rc) return rc;
    if (ops[i].type == CPB200_OP_STEM && (ops[i].flags & CPB200_FLAG_TC)) {
      if (!cpb::stem_tc_eligible(ops[i])) return cpb::fail(CPB200_ERR_ARG, "op %d: shape not supported by the tensor-core stem", i);
    } else if (cpb::sp_eligible(ops[i])) {
      // small-channel 3x3 conv: SIMT-fed wgmma kernel, nothing to prepare (csrc/net_tc_sp.cu)
    } else if (ops[i].flags & CPB200_FLAG_TC) {
      rc = cpb::tc_prepare_op(ops[i]);
      if (rc) return rc;
    }
  }
  return CPB200_OK;
}

extern "C" int cpb200_release_ops(cpb200_op *ops, int n) {
  if (!ops) return CPB200_OK;
  for (int i = 0; i < n; ++i)
    if (ops[i].tc) cpb::tc_release_op(ops[i]);
  return CPB200_OK;
}

extern "C" int cpb200_run_ops(const cpb200_op *ops, int n, void *stream) {
  if (!ops || n < 0) return cpb::fail(CPB200_ERR_ARG, "run_ops: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  for (int i = 0; i < n; ++i) {
    int rc;
    if (!(ops[i].flags & CPB200_FLAG_TC)) rc = cpb::run_op_simt_dispatch(ops[i], st);
    else if (ops[i].type == CPB200_OP_STEM) rc = cpb::stem_tc_run(ops[i], st);
    else if (!ops[i].tc && cpb::sp_eligible(ops[i])) rc = cpb::sp_run(ops[i], st);
    else rc = cpb::tc_run_op(ops[i], st);
    if (rc) return rc;
  }
  return CPB200_OK;
}
