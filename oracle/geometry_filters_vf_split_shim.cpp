// TEST INFRASTRUCTURE: the UNMODIFIED src/utils/vf_split.cpp, included where it lies under $(REF): vf_split for the
// two split shims.
#include "utils/vf_split.cpp"
