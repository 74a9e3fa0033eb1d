// The emulated launchers of nvl_emu_launch.cpp with a datatype table that adds INT128 / UINT128 to its representative subset: the
// tl/nvl plugin that tests/hostemu_int128_worker.py drives (tests/emu/build_hostemu_int128.sh).  The prelude is included first, so
// the kernel sources see the table under its own name, and nvl_emu_launch.cpp's table is compiled under another one.
#define NVL_EMU_LAUNCHERS 1
#include "nvl_emu_prelude.h"

#define nvl_rows nvl_rows_subset
#include "nvl_emu_launch.cpp"
#undef nvl_rows

const nvl_dt_row *const nvl_rows[NVL_DT_LAST] = {
    nvl_rows_subset[NVL_DT_I8], nvl_rows_subset[NVL_DT_I16], nvl_rows_subset[NVL_DT_I32], nvl_rows_subset[NVL_DT_I64],
    nvl_rows_subset[NVL_DT_U8], nvl_rows_subset[NVL_DT_U16], nvl_rows_subset[NVL_DT_U32], nvl_rows_subset[NVL_DT_U64],
    nvl_rows_subset[NVL_DT_F16], nvl_rows_subset[NVL_DT_F32], nvl_rows_subset[NVL_DT_F64], nvl_rows_subset[NVL_DT_BF16],
    nvl_rows_subset[NVL_DT_C64], nvl_rows_subset[NVL_DT_C128], nullptr, &nvl_row_of<nvl_i128>, &nvl_row_of<nvl_u128>};
static_assert(NVL_DT_F128 == 14 && NVL_DT_U128 + 1 == NVL_DT_LAST, "the table above lists every datatype of nvl_kernels.h");
