// Global handle objects of the MPI C API + small helpers
#include <faabric/mpi/MpiMessage.h>
#include <faabric/mpi/mpi.h>

#include <cstdlib>
#include <cstring>
#include <stdexcept>

struct faabric_communicator_t faabric_comm_world = { .id = FAABRIC_COMM_WORLD };
struct faabric_communicator_t faabric_comm_null = { .id = FAABRIC_COMM_NULL };

struct faabric_datatype_t faabric_type_int8 = { .id = FAABRIC_INT8, .size = sizeof(int8_t) };
struct faabric_datatype_t faabric_type_int16 = { .id = FAABRIC_INT16, .size = sizeof(int16_t) };
struct faabric_datatype_t faabric_type_int32 = { .id = FAABRIC_INT32, .size = sizeof(int32_t) };
struct faabric_datatype_t faabric_type_int = { .id = FAABRIC_INT, .size = sizeof(int) };
struct faabric_datatype_t faabric_type_int64 = { .id = FAABRIC_INT64, .size = sizeof(int64_t) };
struct faabric_datatype_t faabric_type_uint8 = { .id = FAABRIC_UINT8, .size = sizeof(uint8_t) };
struct faabric_datatype_t faabric_type_uint16 = { .id = FAABRIC_UINT16, .size = sizeof(uint16_t) };
struct faabric_datatype_t faabric_type_uint32 = { .id = FAABRIC_UINT32, .size = sizeof(uint32_t) };
struct faabric_datatype_t faabric_type_uint = { .id = FAABRIC_UINT, .size = sizeof(unsigned int) };
struct faabric_datatype_t faabric_type_uint64 = { .id = FAABRIC_UINT64, .size = sizeof(uint64_t) };
struct faabric_datatype_t faabric_type_long = { .id = FAABRIC_LONG, .size = sizeof(long) };
struct faabric_datatype_t faabric_type_long_long = { .id = FAABRIC_LONG_LONG, .size = sizeof(long long) };
struct faabric_datatype_t faabric_type_long_long_int = { .id = FAABRIC_LONG_LONG_INT, .size = sizeof(long long int) };
struct faabric_datatype_t faabric_type_float = { .id = FAABRIC_FLOAT, .size = sizeof(float) };
struct faabric_datatype_t faabric_type_double = { .id = FAABRIC_DOUBLE, .size = sizeof(double) };
// {double, int} with natural padding
struct faabric_datatype_t faabric_type_double_int = { .id = FAABRIC_DOUBLE_INT, .size = 16 };
struct faabric_datatype_t faabric_type_char = { .id = FAABRIC_CHAR, .size = sizeof(char) };
struct faabric_datatype_t faabric_type_c_bool = { .id = FAABRIC_C_BOOL, .size = sizeof(bool) };
struct faabric_datatype_t faabric_type_byte = { .id = FAABRIC_BYTE, .size = 1 };
struct faabric_datatype_t faabric_type_null = { .id = FAABRIC_DATATYPE_NULL, .size = 0 };
struct faabric_datatype_t faabric_type_half = { .id = FAABRIC_HALF, .size = 2 };
struct faabric_datatype_t faabric_type_bfloat16 = { .id = FAABRIC_BFLOAT16, .size = 2 };
struct faabric_datatype_t faabric_type_float_int = { .id = FAABRIC_FLOAT_INT, .size = 8 };
struct faabric_datatype_t faabric_type_2int = { .id = FAABRIC_2INT, .size = 8 };
struct faabric_datatype_t faabric_type_long_int = { .id = FAABRIC_LONG_INT, .size = 16 };

struct faabric_info_t faabric_info_null = { .id = FAABRIC_INFO_NULL };
int faabric_unweighted = 0;
int faabric_weights_empty = 0;
struct faabric_info_t faabric_info_device = { .id = FAABRIC_INFO_DEVICE };

struct faabric_op_t faabric_op_max = { .id = FAABRIC_OP_MAX };
struct faabric_op_t faabric_op_min = { .id = FAABRIC_OP_MIN };
struct faabric_op_t faabric_op_sum = { .id = FAABRIC_OP_SUM };
struct faabric_op_t faabric_op_prod = { .id = FAABRIC_OP_PROD };
struct faabric_op_t faabric_op_land = { .id = FAABRIC_OP_LAND };
struct faabric_op_t faabric_op_lor = { .id = FAABRIC_OP_LOR };
struct faabric_op_t faabric_op_band = { .id = FAABRIC_OP_BAND };
struct faabric_op_t faabric_op_bor = { .id = FAABRIC_OP_BOR };
struct faabric_op_t faabric_op_maxloc = { .id = FAABRIC_OP_MAXLOC };
struct faabric_op_t faabric_op_minloc = { .id = FAABRIC_OP_MINLOC };
struct faabric_op_t faabric_op_null = { .id = FAABRIC_OP_NULL };
struct faabric_op_t faabric_op_lxor = { .id = FAABRIC_OP_LXOR };
struct faabric_op_t faabric_op_bxor = { .id = FAABRIC_OP_BXOR };
struct faabric_op_t faabric_op_replace = { .id = FAABRIC_OP_REPLACE };
struct faabric_op_t faabric_op_no_op = { .id = FAABRIC_OP_NO_OP };

struct faabric_datatype_t* getFaabricDatatypeFromId(int datatypeId)
{
#define FAABRIC_MPI_TYPE_CASE(name, num, var)                                  \
    case num:                                                                  \
        return &var;
    switch (datatypeId) {
        FAABRIC_MPI_DATATYPES(FAABRIC_MPI_TYPE_CASE)
        default:
            return nullptr;
    }
#undef FAABRIC_MPI_TYPE_CASE
}

namespace faabric::mpi {

void serializeMpiMsg(std::vector<uint8_t>& buffer, const MpiMessage& msg)
{
    buffer.resize(msgSize(msg));
    memcpy(buffer.data(), &msg, sizeof(MpiMessage));
    size_t payload = payloadSize(msg);
    if (payload > 0 && msg.buffer != nullptr) {
        memcpy(buffer.data() + sizeof(MpiMessage), msg.buffer, payload);
    }
}

void parseMpiMsg(const std::vector<uint8_t>& bytes, MpiMessage* msg)
{
    if (bytes.size() < sizeof(MpiMessage)) {
        throw std::runtime_error("MPI message shorter than its header");
    }
    memcpy(msg, bytes.data(), sizeof(MpiMessage));
    size_t payload = bytes.size() - sizeof(MpiMessage);
    if (payload != payloadSize(*msg)) {
        throw std::runtime_error("MPI message payload size mismatch");
    }
    if (payload == 0) {
        msg->buffer = nullptr;
        return;
    }
    msg->buffer = malloc(payload);
    memcpy(msg->buffer, bytes.data() + sizeof(MpiMessage), payload);
}

}
