/* include/compat/crt_core.h -- lets the reference's unmodified drivers (crt_main.c,
 * extra/video_convert.c: `#include "crt_core.h"`) pick up this library's interface instead of
 * the reference header.  Put this directory first on the include path; see INTEGRATION.md. */
#include "../crt_b200.h"
