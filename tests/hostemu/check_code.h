// check_code.h — TEST INFRASTRUCTURE ONLY: the status an emu entry returns for a check of ggml_b200/csrc/b200_op_checks.h.  It is the
// launcher's status, except that a refusal without a reason returns 1, so that the tests catch a check that refuses without saying why.
#pragma once
#include "../../ggml_b200/csrc/b200_op_checks.h"

inline int code(const b200::op_check & r) { return r.ok() || r.reason ? r.code : 1; }
