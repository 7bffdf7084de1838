// lightctr_b200/csrc/loader.h -- the host parser of libffm text (loader.cpp), for the device parser's fallback (text.cu).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

namespace lctr {

// CSR arrays of parsed text.  Id = uint32_t: ids >= 2^32 are an error (the dense tables are indexed by them);
// Id = uint64_t: ids keep the full %zu width (keyed mode hashes them into rows).
template <typename Id>
struct Parsed {
    std::vector<int64_t> row_ptr{0};
    std::vector<Id> ids;
    std::vector<uint16_t> fields;
    std::vector<float> vals;
    std::vector<int32_t> labels;
    uint64_t feature_cnt = 0, field_cnt = 0;
};

// One line of FM_Algo_Abst::loadDataRow (fm_algo_abst.h:84-104): line[len] must be '\0' (len excludes the '\n').  Its
// label (if one parses) and entries are appended to out; a row is closed when it has entries.  val / nchar: the state
// the reference's loop carries from token to token and from line to line (a two-field token keeps both).  1 at a field
// >= 2^16, with the token's ids in *bad_fid / *bad_field; the line's entries up to it are appended.
int parse_line(const char* line, size_t len, Parsed<uint64_t>& out, float& val, int& nchar, uint64_t* bad_fid,
               uint64_t* bad_field);

}  // namespace lctr
