// window.cuh — the host side of the window functions (window.cu) that GpuWindowExec (exec.cu) drives.
#pragma once
#include "common.cuh"

namespace b2 {

struct WinFn {
  b2_window_spec s;
  int frame;         // FR_*
  int in_dtype = 0;  // input column type (0 for functions without a column)
};

struct WindowPlan {
  std::vector<int32_t> part;
  std::vector<b2_order_by_arg> order;
  std::vector<WinFn> fns;
  int mode = 1;   // 1 running only, 2 a RANGE running frame, 3 a frame that needs the whole partition (LEAD / LAG, RANGE value offsets)
  // P and F: how many rows before (pre) and after (post) a row its frame or LEAD / LAG source can reach.  bounded: every function
  // is ranking, LEAD / LAG or a ROWS frame with a finite upper bound, and P + F > 0; such a plan streams with context rows
  int64_t pre = 0, post = 0;
  bool bounded = false;
};

// What a chunk leaves to the next one: its last row (the boundary of row 0) and every function's state at that row
struct WindowCarry {
  Table* last = nullptr;
  std::vector<DevBuf> state;   // [0] ranking, then one per function (empty where it has none)
  // FIRST / LAST / NTH_VALUE, indexed as state (whose entry is then the int64 count of the open partition's rows so far that
  // count): the one-row column of the value a continuing frame resolves to, or null
  std::vector<Column*> value;
  ~WindowCarry() {
    if (last) table_release(last);
    for (Column* c : value) if (c) col_release(c);
  }
};

// checks the specs and classifies their frames (B2_ERR_INVALID / B2_ERR_UNSUPPORTED); bind_window checks the columns of a batch
WindowPlan make_window_plan(const int32_t* part_cols, int nparts, const b2_order_by_arg* order, int norder, const b2_window_spec* specs, int nspecs);
void bind_window(WindowPlan& p, const Table* t);
// the functions over one chunk of sorted rows, continuing from (and then replacing) the carry when one is given
Table* window_chunk(WindowPlan& p, const Table* t, WindowCarry* carry);
// the functions only, over rows [lo, hi) of `t` (the rows around them are context and look-ahead), continuing from the carry;
// on success the carry becomes the one at row carry_row (-1: it stays as it was)
Table* window_chunk_rows(WindowPlan& p, const Table* t, WindowCarry* carry, int64_t lo, int64_t hi, int64_t carry_row);
// the columns of the input that `p` reads, in the order of a table `over_read` (p with its column indexes remapped) reads them
std::vector<int> window_read_columns(const WindowPlan& p, WindowPlan* over_read);
// the last row of `t` that starts a partition (mask 1) or a peer group (mask 2), row 0 compared with `last`; -1 when none
int64_t window_last_start(const WindowPlan& p, const Table* t, const Table* last, uint8_t mask);

}  // namespace b2
