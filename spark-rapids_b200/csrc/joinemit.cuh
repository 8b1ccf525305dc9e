// joinemit.cuh — the FK -> PK join that writes its output rows from the filter-probe kernel (join.cu) instead of gathering
// them through maps; driven by GpuShuffledHashJoinExec (exec.cu).
#pragma once
#include "common.cuh"

namespace b2 {

struct Program;

// The build columns the emitting probe writes, packed row-major: `width` bytes per build row (8 or 16; 0 = no build
// columns), column k at byte `off[k]` of its row
// Rows are in build row order, or, for a direct table, in the table's rank order (one row per non-NULL key, ascending keys):
// the order in which the probe of `table` finds them.
struct JoinPayload {
  DevBuf packed;
  int width = 0;
  std::vector<int> dtype, scale, off;
  b2_handle table = 0;      // the hash table it was packed for
  bool rank_order = false;
};
// packs columns `cols` of `build` (the table hash table `ht` was built over) into `pl`, in the order `ht` needs.  False: they
// do not qualify (more than 4 columns or 16 bytes, a nullable or STRING column).  Throws B2_ERR_OOM when the array cannot be
// allocated.
bool join_pack_payload(b2_handle ht, const Table* build, const std::vector<int>& cols, JoinPayload& pl);
// The filter `prog` below the stream side and the INNER probe of `batch` in one kernel (join_probe_pred's fast path), writing
// the rows [stream_cols of batch ++ payload columns] into columns of `cap` rows.  *total_out = matches, *npass_out = rows
// that passed the filter; *out = the output when total <= cap (otherwise untouched: the batch must be joined through the
// maps).  False: not applicable (nothing launched): the fast path does not apply, or a stream column is nullable, wider
// than 8 bytes, or one of more than 4.
bool join_probe_pred_emit(b2_handle ht, const Table* batch, int key_col, const Program* prog, const std::vector<int>& stream_cols,
                          const JoinPayload& pl, int64_t cap, Table** out, int64_t* total_out, int64_t* npass_out);

}  // namespace b2
